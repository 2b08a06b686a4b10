"""CPU: the perturbation chart's oracle (oracle/pgo_perturb_oracle.py; include/d2pgo.h d2pgo_set_chart) against the reference's own
RelPoseFactorPerturbAD and GravityPriorPerturbAD (live through oracle/_ref/libd2ref_gravity.so and frozen in
tests/golden/ref_perturb.npz), in both branches of quatfromRotationVector; the converged chart solve against the reference's
objective; the ceres-LM trace in the chart; the node's persistent state; the ABI."""
import ctypes as C
import os

import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pgo_ceres_lm_oracle as co
from oracle import pgo_perturb_oracle as po
from oracle import ref_gravity as ref
from oracle.pgo_gravity_oracle import ego_gravity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_perturb.npz")
LIVE = pytest.mark.skipif(not ref.available(), reason="reference gravity library not built")
MAGNITUDES = (0.0, 1e-6, 5e-3, 0.0099, 0.0101, 0.1, 1.0, 3.0)   # |theta|: both sides of the 1e-2 ball, away from its edge
PER_MAGNITUDE = 32
MIXED = ((5e-3, 0.5), (0.5, 5e-3), (0.0, 1.0), (0.0101, 0.0099))   # (|theta_a|, |theta_b|): one endpoint in the ball, one out
PER_MIXED = 16


def _unit(v):
    return v / np.linalg.norm(v)


def reference_cases(seed=0):
    """Seeded inputs: PER_MAGNITUDE per |theta| of MAGNITUDES (theta_b of the same branch as theta_a), then PER_MIXED per pair of
    MIXED (the two endpoints in different branches): attitudes q_a0, q_b0, states a, b = [p, theta], a relative-pose edge with a
    full non-symmetric S6, an (unnormalised) ego pose and a full S3."""
    rng = np.random.default_rng(seed)
    out = {k: [] for k in ("qa", "qb", "a", "b", "rel", "S6", "ego", "S3")}
    pairs = [(m, None) for m in MAGNITUDES for _ in range(PER_MAGNITUDE)] + [p for p in MIXED for _ in range(PER_MIXED)]
    for m, mb in pairs:
        if mb is None:
            mb = m * rng.uniform(0.5, 0.99) if 0.0 < m < 1e-2 else m
        out["qa"].append(_unit(rng.normal(size=4))); out["qb"].append(_unit(rng.normal(size=4)))
        out["a"].append(np.r_[rng.normal(0, 5, 3), m * _unit(rng.normal(size=3))])
        out["b"].append(np.r_[rng.normal(0, 5, 3), mb * _unit(rng.normal(size=3))])
        out["rel"].append(np.r_[rng.normal(0, 2, 3), _unit(rng.normal(size=4))])
        out["S6"].append(20.0 * np.eye(6) + 5.0 * rng.normal(size=(6, 6)))
        out["ego"].append(np.r_[rng.normal(0, 5, 3), _unit(rng.normal(size=4)) * rng.uniform(0.5, 2.0)])
        out["S3"].append(10.0 * np.eye(3) + 3.0 * rng.normal(size=(3, 3)))
    return {k: np.array(v) for k, v in out.items()}


def reference_outputs(c):
    """The reference functors on reference_cases (what tests/golden/make_ref_perturb_golden.py freezes)."""
    out = {k: [] for k in ("r", "Ja", "Jb", "rg", "Jg")}
    for k in range(len(c["a"])):
        r, Ja, Jb = ref.relpose_perturb_eval(c["rel"][k], c["S6"][k], c["qa"][k], c["qb"][k], c["a"][k], c["b"][k])
        rg, Jg = ref.gravity_prior_eval(c["ego"][k], c["S3"][k], c["qa"][k], c["a"][k])
        for n, v in zip(("r", "Ja", "Jb", "rg", "Jg"), (r, Ja, Jb, rg, Jg)):
            out[n].append(v)
    return {k: np.array(v) for k, v in out.items()}


def oracle_outputs(c):
    r, Ja, Jb = po.relpose_eval(c["a"], c["b"], c["qa"], c["qb"], c["rel"], c["S6"])
    rg, Jg = po.gravity_eval(c["a"], c["qa"], ego_gravity(c["ego"]), c["S3"])
    return dict(r=r, Ja=Ja, Jb=Jb, rg=rg, Jg=Jg)


def check_outputs(got, want, r_tol=1e-13, j_tol=1e-12):
    """residuals within r_tol (absolute, per case scaled by max(1, |r|)); Jacobians within j_tol relative to max(1, |J|)"""
    for k in ("r", "rg"):
        err = np.abs(got[k] - want[k]).max(axis=1) / np.maximum(1.0, np.abs(want[k]).max(axis=1))
        assert err.max() <= r_tol, (k, err.max(), int(err.argmax()))
    for k in ("Ja", "Jb", "Jg"):
        err = np.abs(got[k] - want[k]).max(axis=(1, 2)) / np.maximum(1.0, np.abs(want[k]).max(axis=(1, 2)))
        assert err.max() <= j_tol, (k, err.max(), int(err.argmax()))


def test_cases_cover_both_branches():
    c = reference_cases()
    assert len(c["a"]) >= 200
    n = np.linalg.norm(c["a"][:, 3:], axis=1); nb = np.linalg.norm(c["b"][:, 3:], axis=1)
    assert (n < 1e-2).sum() >= 100 and (n >= 1e-2).sum() >= 100
    assert np.abs(n - 1e-2).min() > 1e-12 and np.abs(nb - 1e-2).min() > 1e-12   # away from the ball's edge
    assert ((n < 1e-2) != (nb < 1e-2)).sum() >= 32                             # edges across the two branches


@LIVE
def test_oracle_matches_the_reference_functors():
    c = reference_cases()
    check_outputs(oracle_outputs(c), reference_outputs(c))


def test_oracle_matches_the_frozen_reference():
    g = np.load(GOLD)
    c = {k[5:]: g[k] for k in g.files if k.startswith("case_")}
    for k, v in reference_cases().items():
        np.testing.assert_array_equal(c[k], v)
    check_outputs(oracle_outputs(c), {k: g[k] for k in ("r", "Ja", "Jb", "rg", "Jg")})


def test_ball_branch_is_unnormalised():
    dq, J = po.quat_from_rotation_vector(np.array([3e-3, -4e-3, 0.0]))
    np.testing.assert_array_equal(dq, [1.5e-3, -2e-3, 0.0, 1.0])
    np.testing.assert_array_equal(J, np.vstack([0.5 * np.eye(3), np.zeros(3)]))
    dq, _ = po.quat_from_rotation_vector(np.array([0.0, 0.0, 0.0101]))
    assert abs(np.linalg.norm(dq) - 1.0) < 1e-15 and abs(dq[3] - np.cos(0.00505)) < 1e-16


def chart_graph(seed=11, n=30, loops=60, priors=False, theta=0.05):
    """a small graph entered into the chart (q_init = the initial attitudes), then a seeded theta of norm `theta` on every free
    pose on top of it, so the starting attitudes are the initial ones perturbed"""
    g = pgo.make_pose_graph(seed=seed, n_agents=2, poses_per_agent=n, loops=loops)
    x, qi = po.enter(g["init"])
    rng = np.random.default_rng(seed)
    th = rng.normal(size=(len(x), 3)); th *= theta / np.linalg.norm(th, axis=1, keepdims=True)
    th[np.asarray(g["fixed"]) != 0] = 0.0
    x[:, 3:] = th
    ego = pgo.make_gravity_case(g, seed=2)["ego"] if priors else None
    n_p = len(x)
    pri = (np.arange(n_p), ego, np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (n_p, 1, 1))) if priors else ()
    prob = po.ChartProblem(x, qi, g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], *pri)
    return g, prob, ego


def reference_gradient(prob, x, g, ego):
    """J^T r over the free 6-vectors assembled from the reference's own functors"""
    n = len(x); gr = np.zeros((n, 6)); qi = prob.qinit
    for e in range(len(g["ea"])):
        a, b = g["ea"][e], g["eb"][e]
        r, Ja, Jb = ref.relpose_perturb_eval(g["rel"][e], g["sqrt_info"][e], qi[a], qi[b], x[a], x[b])
        gr[a] += Ja.T @ r; gr[b] += Jb.T @ r
    if ego is not None:
        for i in range(n):
            r, J = ref.gravity_prior_eval(ego[i], pgo.GRAVITY_SQRT_INFO * np.eye(3), qi[i], x[i])
            gr[i] += J.T @ r
    return gr[np.asarray(g["fixed"]) == 0]


@LIVE
@pytest.mark.parametrize("priors", [False, True])
def test_converged_chart_solve_is_a_stationary_point_of_the_reference_objective(priors):
    g, prob, ego = chart_graph(priors=priors)
    x, costs = po.solve_chart(prob)
    g0 = np.abs(reference_gradient(prob, prob.x0, g, ego)).max()
    g1 = np.abs(reference_gradient(prob, x, g, ego)).max()
    assert g1 <= 1e-8 * g0, (g1, g0)
    assert costs[-1] < costs[0]


def test_ceres_lm_trace_in_the_chart():
    _, prob, _ = chart_graph(seed=5, priors=True)
    # the first step against a long-double solve of (J^T J + diag(mu)) dx = -g
    r, J, d = prob.system(prob.x0)
    scale = co.jacobi_scale(d)
    mu = co.damping(d, scale, 1e4)
    dx = co.lm_step(J, r, mu)
    A = (J.T @ J).toarray().astype(np.longdouble) + np.diag(mu.astype(np.longdouble)); b = -(J.T @ r).astype(np.longdouble)
    res = A @ dx.astype(np.longdouble) - b
    assert float(np.abs(res).max()) <= 1e-9 * float(np.abs(b).max())
    # m = C - |r + J dx|^2 / 2
    m = co.model_cost_change(J, r, dx)
    f = r + J @ dx
    assert abs(m - (0.5 * r @ r - 0.5 * f @ f)) <= 1e-9 * abs(m)
    # exactly k iterations
    for k in (1, 3, 7):
        _, tr, rep = co.ceres_lm_solve(prob, max_num_iterations=k, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
        assert len(tr) == k and rep["reason"] == co.MAX_ITERATIONS
    # the gradient and parameter tests run on the 6-vectors
    x = prob.x0
    gvec = prob.gradient(x)
    assert co.gradient_max_norm(prob, x, gvec) == np.abs(x[prob.free] - (x[prob.free] + (-gvec.reshape(-1, 6)))).max()
    assert co.ambient_norm(prob, x) == float(np.linalg.norm(x[prob.free]))
    _, tr, rep = co.ceres_lm_solve(prob, gradient_tolerance=10 * co.gradient_max_norm(prob, x, gvec))
    assert rep["reason"] == co.GRADIENT and not tr


def test_node_state_persists_across_solves():
    g = pgo.make_pose_graph(seed=3, n_agents=2, poses_per_agent=20, loops=30)
    ids = np.asarray(g["ids"]); n = len(ids)
    first = np.arange(n) < n - 6                              # the last six poses arrive before the second solve
    st = po.NodeState(ids[first], g["init"][first])
    x0, q0 = st.arrays(ids[first])
    np.testing.assert_array_equal(x0[:, 3:], 0.0)
    np.testing.assert_allclose(np.linalg.norm(q0, axis=1), 1.0, rtol=0, atol=1e-15)
    sel = first[g["ea"]] & first[g["eb"]]
    remap = -np.ones(n, int); remap[first] = np.arange(first.sum())
    st.solve(ids[first], np.asarray(g["fixed"])[first], remap[g["ea"][sel]], remap[g["eb"][sel]], g["rel"][sel], g["sqrt_info"][sel], po.solve_chart)
    x1, q1 = st.arrays(ids[first])
    np.testing.assert_array_equal(q1, q0)                     # a solve moves [p, theta] only
    moved = g["init"].copy(); moved[:, :3] += 100.0          # set_poses: present ids ignore their given pose
    st.set_poses(ids, moved)
    x2, q2 = st.arrays(ids)
    np.testing.assert_array_equal(x2[first], x1); np.testing.assert_array_equal(q2[first], q1)
    xn, qn = po.enter(moved[~first])
    np.testing.assert_array_equal(x2[~first], xn); np.testing.assert_array_equal(q2[~first], qn)
    # rotation initialisation replaces q_init only
    after = st.poses(ids); after[:, 3:7] = np.roll(after[:, 3:7], 1, axis=0)
    st.rot_init(ids, after)
    x3, q3 = st.arrays(ids)
    np.testing.assert_array_equal(x3, x2)
    np.testing.assert_allclose(q3, after[:, 3:7], rtol=0, atol=1e-15)


def test_abi_chart():
    from d2slam_b200 import build, solver
    build.build()
    lib = solver.lib()
    for n in ("d2pgo_set_chart", "d2pgo_set_perturb", "d2pgo_get_perturb"):
        assert hasattr(lib, n) and n in pgo.PGO_EXPORTED
    assert pgo.CHARTS == {"retraction": 0, "perturb": 1}
    hdr = open(os.path.join(ROOT, "include", "d2pgo.h")).read()
    assert "D2PGO_CHART_RETRACTION = 0, D2PGO_CHART_PERTURB = 1" in hdr
    # null handles are refused before any device work
    assert lib.d2pgo_set_chart(None, C.c_int32(1), C.c_int32(0), None, None) == 1
    assert lib.d2pgo_set_perturb(None, C.c_int32(0), None, None) == 1
    assert lib.d2pgo_get_perturb(None, C.c_int32(0), None, None, None) == 1
