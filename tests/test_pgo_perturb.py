"""GPU: the pose graph in d2pgo's perturbation chart (include/d2pgo.h d2pgo_set_chart) against its CPU oracle
(oracle/pgo_perturb_oracle.py) and the reference functors frozen in tests/golden/ref_perturb.npz: the factor records in both
branches of quatfromRotationVector, ceres-LM traces, the restated loop on both linear solvers, the node's solve sequence,
reproducibility and the time budget, and the refusals."""
import os

import numpy as np
import pytest

from d2slam_b200 import pgo, solver
from oracle import pgo_arock_oracle as ao
from oracle import pgo_ceres_lm_oracle as co
from oracle import pgo_perturb_oracle as po

import test_pgo_arock as tpa
import test_pgo_ceres_lm as tcl
import test_pgo_perturb_oracle as tpo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_perturb.npz")


def chart_device(g, prob, ego=None, linear_solver="sparse_cholesky", **kw):
    """a handle holding g's poses and edges in the chart, at prob's states and q_init"""
    s = pgo.PgoSolver(linear_solver=linear_solver, **kw)
    s.set_poses(g["ids"], g["init"], g["fixed"])
    s.set_chart("perturb", g["ids"], prob.qinit)
    s.set_perturb(g["ids"], prob.x0)
    s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    if ego is not None:
        s.add_gravity_priors(g["ids"], ego)
    return s


def max_rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(1.0, np.abs(np.asarray(b)).max()))


@pytest.mark.gpu
def test_debug_hooks_match_the_reference_functors():
    gd = np.load(GOLD)
    c = {k[5:]: gd[k] for k in gd.files if k.startswith("case_")}
    K = len(c["a"])
    ids = np.arange(2 * K, dtype=np.int64)
    poses = np.zeros((2 * K, 7)); poses[0::2, 3:] = c["qa"]; poses[1::2, 3:] = c["qb"]
    q = np.zeros((2 * K, 4)); q[0::2] = c["qa"]; q[1::2] = c["qb"]
    x = np.zeros((2 * K, 6)); x[0::2] = c["a"]; x[1::2] = c["b"]
    s = pgo.PgoSolver()
    s.set_poses(ids, poses)
    s.set_chart("perturb", ids, q)
    s.set_perturb(ids, x)
    s.add_edges(ids[0::2], ids[1::2], c["rel"], c["S6"])
    s.add_gravity_priors(ids[0::2], c["ego"], c["S3"])
    e = s.debug_edges(); gp = s.debug_gravity_priors()
    s.close()
    orc = tpo.oracle_outputs(c)
    for want in ({k: gd[k] for k in ("r", "Ja", "Jb", "rg", "Jg")}, orc):
        for k in range(K):   # per case, both branches
            assert max_rel(e[k, :6], want["r"][k]) <= 1e-11, k
            assert max_rel(e[k, 6:42].reshape(6, 6), want["Ja"][k]) <= 1e-11, k
            assert max_rel(e[k, 42:].reshape(6, 6), want["Jb"][k]) <= 1e-11, k
            assert max_rel(gp[k, :3], want["rg"][k]) <= 1e-11, k
            assert max_rel(gp[k, 3:].reshape(3, 6), want["Jg"][k]) <= 1e-11, k


def chart_case(name):
    if name == "bench":
        g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
        x, qi = po.enter(g["init"])
        return g, po.ChartProblem(x, qi, g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"]), None
    return tpo.chart_graph(seed=11 if name == "6dof" else 13, priors=name == "6dof_gravity")


BENCH_WINDOW = 10   # iterations of the bench trace held to 1e-10


def bench_traces_agree(td, to, rep_d, rep_o):
    """The bench graph's 50 ceres iterations.  Every step kind and the termination are equal.  C, C+, m and the radius agree within
    1e-10 over the first BENCH_WINDOW iterations and within 1e-8 over all 50: the radius is the product of one factor per
    accepted step, each a function of rho = (C - C+) / m, so the rounding of every earlier rho accumulates in it (the first
    iteration past 1e-10 is the 16th, at 1.2e-10)."""
    assert len(td["kind"]) == len(to) == 50
    assert list(td["kind"]) == [t["kind"] for t in to]
    assert (pgo.TERMINATIONS[rep_o["type"]], pgo.STOP_REASONS[rep_o["reason"]]) == (rep_d["termination"], rep_d["stop"])
    for f in ("cost", "candidate_cost", "model_cost_change", "radius"):
        o = np.array([t[f] for t in to])
        rel = np.abs(td[f] - o) / np.abs(o)
        assert rel[:BENCH_WINDOW].max() <= 1e-10 and rel.max() <= 1e-8, (f, rel[:BENCH_WINDOW].max(), rel.max(), int(rel.argmax()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof", "6dof_gravity", "bench"])
def test_ceres_lm_trace_matches_the_oracle(name):
    g, prob, ego = chart_case(name)
    cfg = dict() if name == "bench" else dict(function_tolerance=1e-12, max_num_iterations=60)   # bench: ceres' defaults, 50 iterations
    x_o, to, rep_o = co.ceres_lm_solve(prob, **cfg)
    s = chart_device(g, prob, ego)
    s.set_minimizer("ceres_lm", **cfg)
    r = s.solve()
    rep_d = s.minimizer_report(); td = s.debug_minimizer_trace(); x_d, q_d = s.get_perturb(g["ids"])
    s.close()
    if name == "bench":
        bench_traces_agree(td, to, rep_d, rep_o)
    else:
        assert tcl.compare_traces(td, to, rep_d, rep_o) >= 1
    assert tcl.close(r.final_cost, rep_o["final_cost"]) and tcl.close(r.initial_cost, rep_o["initial_cost"])
    np.testing.assert_allclose(q_d, prob.qinit, rtol=0, atol=1e-15)   # the handle normalises q_init again
    assert np.abs(x_d - x_o).max() < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("linear_solver", ["pcg", "sparse_cholesky"])
def test_restated_loop_reaches_the_oracle_optimum(linear_solver):
    g, prob, ego = tpo.chart_graph(seed=17, priors=True)
    x_o, costs = po.solve_chart(prob)
    s = chart_device(g, prob, ego, linear_solver=linear_solver, max_iterations=100, pcg_max_iterations=2000, pcg_tolerance=1e-13,
                     function_tolerance=1e-15)
    r = s.solve()
    x_d, _ = s.get_perturb(g["ids"]); p_d = s.get_poses(g["ids"])
    s.close()
    assert abs(r.final_cost - costs[-1]) <= 1e-10 * costs[-1], (r.final_cost, costs[-1])
    assert np.abs(x_d - x_o).max() < 1e-6
    dp, dr = tcl.tc.pose_diff6(p_d, po.poses_of(x_o, prob.qinit))
    assert dp < 1e-6 and dr < 1e-6


@pytest.mark.gpu
def test_node_solve_sequence_matches_the_oracle():
    g = pgo.make_pose_graph(seed=21, n_agents=1, poses_per_agent=50, loops=60)   # one trajectory: every component holds pose 0
    ids = np.asarray(g["ids"]); n = len(ids); fixed = np.asarray(g["fixed"])
    first = np.arange(n) < n - 8
    sel = first[g["ea"]] & first[g["eb"]]
    cfg = dict(max_num_iterations=50)
    s = pgo.PgoSolver(linear_solver="sparse_cholesky")
    s.set_minimizer("ceres_lm", **cfg)
    s.set_poses(ids[first], g["init"][first], fixed[first])
    s.set_chart("perturb")
    s.add_edges(g["id_a"][sel], g["id_b"][sel], g["rel"][sel], g["sqrt_info"][sel])
    st = po.NodeState(ids[first], g["init"][first])
    before = s.get_poses(ids[first])
    x_before, _ = s.get_perturb(ids[first])
    s.rot_init()
    x_after, q_after = s.get_perturb(ids[first])
    np.testing.assert_array_equal(x_after, x_before)           # rotation initialisation leaves p and theta
    # the reference value: d2pgo_rot_init on a retraction-chart handle holding the composed attitudes
    r = pgo.PgoSolver()
    r.set_poses(ids[first], before, fixed[first])
    r.add_edges(g["id_a"][sel], g["id_b"][sel], g["rel"][sel], g["sqrt_info"][sel])
    r.rot_init()
    after = r.get_poses(ids[first])
    r.close()
    named = np.zeros(first.sum(), bool); named[g["ea"][sel]] = True; named[g["eb"][sel]] = True
    free = named & (fixed[first] == 0)
    assert free.sum() > 10 and np.abs(after[free, 3:] - before[free, 3:]).max() > 1e-3   # the initialisation moves them
    np.testing.assert_allclose(q_after, po.enter(after)[1], rtol=0, atol=1e-15)
    np.testing.assert_allclose(q_after[~free], po.enter(before[~free])[1], rtol=0, atol=1e-15)
    st.rot_init(ids[first], after)
    remap = -np.ones(n, int); remap[first] = np.arange(first.sum())
    s.solve()
    st.solve(ids[first], fixed[first], remap[g["ea"][sel]], remap[g["eb"][sel]], g["rel"][sel], g["sqrt_info"][sel], co.ceres_lm_solve, **cfg)
    # the node's state grows: every pose again (present ones keep their state), every edge
    s.set_poses(ids, g["init"], fixed)
    s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    st.set_poses(ids, g["init"])
    x_d, q_d = s.get_perturb(ids); x_o, q_o = st.arrays(ids)
    assert np.abs(x_d - x_o).max() < 1e-6
    np.testing.assert_allclose(q_d, q_o, rtol=0, atol=1e-15)
    s.solve()
    st.solve(ids, fixed, g["ea"], g["eb"], g["rel"], g["sqrt_info"], co.ceres_lm_solve, **cfg)
    x_d, q_d = s.get_perturb(ids); x_o, q_o = st.arrays(ids)
    s.close()
    assert np.abs(x_d - x_o).max() < 1e-6
    np.testing.assert_allclose(q_d, q_o, rtol=0, atol=1e-15)


@pytest.mark.gpu
def test_reproducible_and_budget_keeps_the_state():
    g, prob, ego = tpo.chart_graph(seed=23, priors=True)
    out = []
    for _ in range(2):
        s = chart_device(g, prob, ego)
        s.set_minimizer("ceres_lm")
        s.solve()
        out.append(s.get_perturb(g["ids"])[0])
        s.close()
    np.testing.assert_array_equal(out[0], out[1])
    s = chart_device(g, prob, ego)
    s.set_minimizer("ceres_lm", max_solver_time_in_seconds=1e-9)
    s.solve()
    assert s.minimizer_report()["stop"] == "time"
    np.testing.assert_array_equal(s.get_perturb(g["ids"])[0], prob.x0)
    s.close()


@pytest.mark.gpu
def test_refusals_keep_nothing():
    g, prob, ego = tpo.chart_graph(seed=29)
    ids = np.asarray(g["ids"])
    s4 = pgo.PgoSolver(pose_dof=4)
    h = pgo.pose_graph_to_4d(g, seed=1)
    s4.set_poses_4d(h["ids"], h["init"], h["fixed"])
    with pytest.raises(RuntimeError, match="rc=5"):
        s4.set_chart("perturb")
    s4.close()
    s = pgo.PgoSolver(linear_solver="sparse_cholesky")
    s.set_poses(ids, g["init"], g["fixed"])
    with pytest.raises(RuntimeError, match="rc=5"):
        s.set_perturb(ids[:1], np.zeros((1, 6)))
    with pytest.raises(RuntimeError, match="rc=5"):
        s.get_perturb(ids[:1])
    for bad_ids, q in ((np.array([10 ** 12]), np.array([[0, 0, 0, 1.0]])), (np.array([10 ** 12]), None), (ids[:1], np.zeros((1, 4))),
                       (ids[:1], np.array([[np.nan, 0, 0, 1.0]]))):
        with pytest.raises(RuntimeError, match="rc=2"):
            s.set_chart("perturb", bad_ids, q)
        np.testing.assert_array_equal(s.get_poses(ids), g["init"])   # still the retraction handle, untouched
    s.set_chart("perturb", ids, prob.qinit)
    s.set_perturb(ids, prob.x0)
    with pytest.raises(RuntimeError, match="rc=2"):
        s.set_perturb(np.array([ids[0], 10 ** 12]), np.zeros((2, 6)))
    with pytest.raises(RuntimeError, match="rc=2"):
        s.set_perturb(ids[:2], np.array([[0, 0, 0, 0, 0, 0], [np.inf, 0, 0, 0, 0, 0]]))
    np.testing.assert_array_equal(s.get_perturb(ids)[0], prob.x0)
    bad = g["init"].copy(); bad[:, 3:] = 0.0
    with pytest.raises(RuntimeError, match="rc=2"):
        s.set_poses(np.r_[ids, 10 ** 12], np.r_[bad, bad[:1]])   # a new id with a zero quaternion
    np.testing.assert_array_equal(s.get_perturb(ids)[0], prob.x0)
    with pytest.raises(RuntimeError, match="rc=5"):
        s.comm_init(bytes(128), 0, 1)
    with pytest.raises(ValueError):
        s.set_chart("exp")
    s.close()
    # a handle with a communicator refuses the chart
    c = pgo.PgoSolver()
    c.set_poses(ids, g["init"], g["fixed"])
    c.comm_init(solver.comm_unique_id(), 0, 1)
    with pytest.raises(RuntimeError, match="rc=5"):
        c.set_chart("perturb")
    np.testing.assert_array_equal(c.get_poses(ids), g["init"])
    c.close()
    # an ARock handle enters the chart before its first step, not after; the distributed rotation initialisation precedes it
    gg = tpa.graph(6)
    sp = pgo.arock_split(gg, 0)
    a = pgo.ArockAgent(sp)
    a.s.set_chart("perturb")
    for call in (lambda: a.s.arock_rot_init_step(), lambda: a.s.arock_rot_receive(1, 0, sp["ids"][:1], np.zeros((1, 9)), sp["poses"][:1])):
        with pytest.raises(RuntimeError, match="rc=5"):
            call()
    a.s.set_chart("retraction")
    a.step()
    with pytest.raises(RuntimeError, match="rc=5"):
        a.s.set_chart("perturb")
    a.close()


@pytest.mark.gpu
def test_debug_steps_solve_the_chart_system():
    g, prob, ego = tpo.chart_graph(seed=31, priors=True)
    r, J, d = prob.system(prob.x0)
    lam = 1e-3
    H = (J.T @ J).toarray() + np.diag(lam * d + 1e-12)
    dx_o = np.linalg.solve(H, -(J.T @ r))
    s = chart_device(g, prob, ego)
    dx_c = s.debug_exact_step(lam)
    dx_p, it, res = s.debug_pcg_step(lam, 5000, 1e-14)
    s.close()
    free = np.asarray(g["fixed"]) == 0
    assert np.all(dx_c[~free] == 0) and np.all(dx_p[~free] == 0)
    assert max_rel(dx_c[free].ravel(), dx_o) <= 1e-8
    assert max_rel(dx_p[free].ravel(), dx_o) <= 1e-8 and res <= 1e-14, (it, res)


@pytest.mark.gpu
def test_arock_in_the_chart_matches_the_oracle_agents():
    """three agents in the chart (ARockPGO in perturb mode) on the ceres minimiser against the oracle's chart agents: poses and
    duals within 1e-6 every round, and the device's proximal records exact to 1e-12 at its own state and duals"""
    gg = tpa.graph(6)
    cfg = tpa.SHIPPED["d435_multi"]
    lm = dict(max_num_iterations=100, function_tolerance=1e-10, parameter_tolerance=1e-12)
    dev = tpa.device_agents(gg, cfg, solver_kw=dict(linear_solver="sparse_cholesky"))
    for a in dev:
        a.s.set_chart("perturb")
        a.s.set_minimizer("ceres_lm", **lm)
    orc = [po.arock_agent(pgo.arock_split(gg, k), lm, **cfg) for k in range(3)]
    for rnd in range(6):
        pgo.arock_run(dev, 1); ao.arock_run(orc, 1)
        for d, o in zip(dev, orc):
            x_d, _ = d.s.get_perturb(d.split["ids"])
            assert np.abs(x_d - o.x).max() < 1e-6, (rnd, d.self_id)
            dp, dr = tcl.tc.pose_diff6(d.poses(), o.poses())
            assert dp < 1e-6 and dr < 1e-6, (rnd, d.self_id, dp, dr)
            dd = d.duals()
            assert sorted(dd) == sorted(o.duals) and dd
            for key, (yl, yr) in dd.items():
                assert np.abs(yl - o.duals[key][0]).max() < 1e-6 and np.abs(yr - o.duals[key][1]).max() < 1e-6, (rnd, key)
            keys = sorted(dd)
            pos = {int(i): k for k, i in enumerate(d.split["ids"])}
            idx = np.array([pos[f] for _, f in keys])
            yr = np.array([dd[k][1] for k in keys])
            rk, Jk = po.prox_eval(x_d[idx], yr, cfg["rho_frame_T"], cfg["rho_frame_theta"])
            terms = d.s.debug_arock_terms(len(keys))
            assert np.abs(terms - np.concatenate([rk, Jk.reshape(len(keys), -1)], axis=1)).max() <= 1e-12, (rnd, d.self_id)
    for a in dev:
        a.s.close()
