"""CPU: the ceres minimiser's oracle (oracle/pgo_ceres_lm_oracle.py) on small hand-built graphs, and its C ABI (symbols, the
defaults d2pgo_default_ceres_lm_config states, struct layouts).  The first damped step against a long-double solve, the model
against C - |r + J dx|^2 / 2 evaluated directly, the trust-region formulas on a scripted rho sequence, the Jacobi scale taken
once, and every stop reason."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from d2slam_b200 import pgo, synth
from oracle import pgo_ceres_lm_oracle as co
from oracle import pgo_lm_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def chain6(n=6, seed=0, noise=0.05, consistent=False, isolated=False):
    """A 6-DoF chain with one loop: odometry between consecutive poses, pose 0 fixed, initial poses perturbed; isolated: one
    more free pose that no edge names (a zero column of J, so H is singular without damping)."""
    rng = np.random.default_rng(seed)
    truth = np.zeros((n, 7)); truth[:, 6] = 1.0
    for i in range(1, n):
        truth[i] = synth.pose_plus(truth[i - 1], np.r_[1.0, 0.2 * rng.normal(size=2), 0.1 * rng.normal(size=3)])
    ea = list(range(n - 1)) + [0]; eb = list(range(1, n)) + [n - 1]
    rel = np.array([pgo.relative_pose(truth[a], truth[b]) for a, b in zip(ea, eb)])
    if not consistent:
        rel[:, :3] += rng.normal(0, 0.05, (len(ea), 3))
    x0 = truth.copy() if consistent else np.array([synth.pose_plus(t, rng.normal(0, noise, 6)) for t in truth])
    x0[0] = truth[0]
    fixed = np.zeros(n, np.uint8); fixed[0] = 1
    S = np.tile(np.eye(6), (len(ea), 1, 1)) * 2.0
    if isolated:
        x0 = np.vstack([x0, x0[1]]); fixed = np.r_[fixed, 0].astype(np.uint8)
    return lo.Problem(x0, fixed, np.array(ea), np.array(eb), rel, S)


def chain4(n=6, seed=1):
    """A 4-DoF chain with one loop whose yaws cross +-pi."""
    rng = np.random.default_rng(seed)
    yaw = pgo.normalize_angle(np.pi - 0.3 + 0.15 * np.arange(n))
    truth = np.c_[np.cumsum(rng.normal(1, 0.1, n)), rng.normal(0, 0.3, n), rng.normal(0, 0.1, n), yaw]
    ea = np.r_[np.arange(n - 1), 0]; eb = np.r_[np.arange(1, n), n - 1]
    rel = np.zeros((len(ea), 4))
    for k, (a, b) in enumerate(zip(ea, eb)):
        c, s = np.cos(-truth[a, 3]), np.sin(-truth[a, 3])
        v = truth[b, :3] - truth[a, :3]
        rel[k] = [c * v[0] - s * v[1], s * v[0] + c * v[1], v[2], pgo.normalize_angle(truth[b, 3] - truth[a, 3])]
    rel += rng.normal(0, 0.03, rel.shape)
    x0 = truth + rng.normal(0, 0.05, truth.shape); x0[:, 3] = pgo.normalize_angle(x0[:, 3]); x0[0] = truth[0]
    fixed = np.zeros(n, np.uint8); fixed[0] = 1
    return lo.Problem(x0, fixed, ea, eb, rel, np.tile(np.eye(4), (len(ea), 1, 1)))


@pytest.mark.parametrize("make", [chain6, chain4])
def test_first_step_equals_a_long_double_solve_and_the_model_its_direct_value(make):
    prob = make()
    x, trace, rep = co.ceres_lm_solve(prob, max_num_iterations=1)
    r, J, d = prob.system(prob.x0)
    s = co.jacobi_scale(d)
    assert np.array_equal(rep["scale"], s)
    mu = co.damping(d, s, 1e4)
    A = (J.T @ J).toarray().astype(np.longdouble) + np.diag(mu.astype(np.longdouble))
    b = -(J.T @ r).astype(np.longdouble)
    ref = np.linalg.solve(A.astype(np.float64), b.astype(np.float64))
    for _ in range(3):   # iterative refinement in long double
        ref = ref + np.linalg.solve(A.astype(np.float64), (b - A @ ref.astype(np.longdouble)).astype(np.float64))
    dx = co.lm_step(J, r, mu)
    assert np.abs(dx - ref).max() <= 1e-12 * np.abs(ref).max()
    m = co.model_cost_change(J, r, dx)
    direct = 0.5 * float(r @ r) - 0.5 * float((r + J @ dx) @ (r + J @ dx))
    assert abs(m - direct) <= 1e-12 * abs(direct)
    assert trace[0]["model_cost_change"] == pytest.approx(m, rel=1e-14)
    assert trace[0]["step_norm"] == pytest.approx(np.linalg.norm(dx), rel=1e-14)


def test_radius_and_decrease_factor_follow_the_formulas():
    lm = co.LmStrategy(1e4, 1e16)
    radius, df = 1e4, 2.0
    for rho in [0.9, 0.5, -1.0, 1e-4, 2.0, 0.999, -5.0, -5.0, -5.0, 0.3]:
        if rho > 1e-3:
            lm.accepted(rho)
            radius = min(radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3), 1e16); df = 2.0
        else:
            lm.rejected()
            radius = radius / df; df = 2.0 * df
        assert lm.radius == pytest.approx(radius, rel=1e-15) and lm.decrease_factor == df
    capped = co.LmStrategy(1e15, 1e16)
    for _ in range(3):
        capped.accepted(1.0)
    assert capped.radius == 1e16


def test_trace_follows_the_trust_region_updates():
    x, trace, rep = co.ceres_lm_solve(chain6(seed=4, noise=0.3), max_num_iterations=30, initial_trust_region_radius=1e-2,
                                      function_tolerance=1e-15, parameter_tolerance=1e-15, gradient_tolerance=1e-15)
    radius, df = 1e-2, 2.0
    for t in trace:
        if t["kind"] == co.ACCEPTED:
            radius = min(radius / max(1.0 / 3.0, 1.0 - (2.0 * t["relative_decrease"] - 1.0) ** 3), 1e16); df = 2.0
            assert t["relative_decrease"] > 1e-3
        elif t["kind"] in (co.REJECTED, co.INVALID):
            radius /= df; df *= 2.0
        assert t["radius"] == pytest.approx(radius, rel=1e-14) and t["decrease_factor"] == df
    assert rep["successful_steps"] + rep["unsuccessful_steps"] == len(trace)


def test_jacobi_scale_is_taken_once():
    prob = chain6(seed=2, noise=0.2)
    calls = []
    orig = co.jacobi_scale
    co.jacobi_scale = lambda d, j=1: calls.append(d.copy()) or orig(d, j)
    try:
        _, trace, rep = co.ceres_lm_solve(prob, max_num_iterations=8)
    finally:
        co.jacobi_scale = orig
    assert len(calls) == 1 and sum(t["kind"] == co.ACCEPTED for t in trace) >= 2
    assert np.array_equal(rep["scale"], orig(prob.system(prob.x0)[2]))


def test_a_consistent_graph_stops_on_the_gradient_at_zero_iterations():
    x, trace, rep = co.ceres_lm_solve(chain6(consistent=True), gradient_tolerance=1e-8)
    assert trace == [] and (rep["type"], rep["reason"]) == (co.CONVERGENCE, co.GRADIENT)
    assert np.array_equal(x, chain6(consistent=True).x0)


@pytest.mark.parametrize("k", [0, 1, 3])
def test_max_num_iterations_gives_exactly_k_iterations(k):
    _, trace, rep = co.ceres_lm_solve(chain6(seed=5, noise=0.3), max_num_iterations=k, function_tolerance=0.0,
                                      parameter_tolerance=0.0, gradient_tolerance=0.0)
    assert len(trace) == k and (rep["type"], rep["reason"]) == (co.NO_CONVERGENCE, co.MAX_ITERATIONS)


def test_every_stop_reason_is_reachable():
    reasons = {}
    _, _, r = co.ceres_lm_solve(chain6(consistent=True)); reasons[co.GRADIENT] = r
    _, _, r = co.ceres_lm_solve(chain6(seed=6), parameter_tolerance=1.0); reasons[co.PARAMETER] = r
    _, _, r = co.ceres_lm_solve(chain6(seed=6), function_tolerance=0.9, parameter_tolerance=0.0); reasons[co.FUNCTION] = r
    _, _, r = co.ceres_lm_solve(chain6(seed=6), min_relative_decrease=1e6, min_trust_region_radius=1e2,
                                parameter_tolerance=0.0, function_tolerance=0.0); reasons[co.MIN_RADIUS] = r
    _, _, r = co.ceres_lm_solve(chain6(seed=6), max_num_iterations=2, function_tolerance=0.0); reasons[co.MAX_ITERATIONS] = r
    with np.errstate(all="ignore"), pytest.warns(Warning):   # scipy warns of the singular matrix
        _, _, r = co.ceres_lm_solve(chain6(seed=6, isolated=True), min_lm_diagonal=1e-300, max_lm_diagonal=1e-300,
                                    initial_trust_region_radius=1e300, max_trust_region_radius=1e300, jacobi_scaling=0,
                                    max_num_consecutive_invalid_steps=0)
    reasons[co.INVALID_STEPS] = r
    for why, rep in reasons.items():
        assert rep["reason"] == why, (why, rep["reason"])
        want = co.FAILURE if why == co.INVALID_STEPS else co.CONVERGENCE if why != co.MAX_ITERATIONS else co.NO_CONVERGENCE
        assert rep["type"] == want


def test_parameter_and_function_stops_return_x_not_the_candidate():
    prob = chain6(seed=7)
    for kw in (dict(parameter_tolerance=1.0), dict(function_tolerance=0.99, parameter_tolerance=0.0)):
        x, trace, rep = co.ceres_lm_solve(prob, **kw)
        assert len(trace) == 1 and trace[0]["kind"] == co.CONVERGED and np.array_equal(x, prob.x0)
        assert rep["unsuccessful_steps"] == 1 and rep["final_cost"] == rep["initial_cost"]


def test_default_settings_reach_the_gauss_newton_optimum():
    prob = chain6(seed=8, noise=0.2)
    x, _, rep = co.ceres_lm_solve(prob, max_num_iterations=200, function_tolerance=1e-15, parameter_tolerance=1e-15)
    y, _, _ = lo.lm_solve(prob, max_iterations=100, lambda0=1e-6, function_tolerance=1e-15)
    assert np.abs(x - y).max() < 1e-7 and rep["type"] == co.CONVERGENCE


# ------------------------------------------------------------------------------------------------ the C ABI
def test_minimizer_symbols_and_config_defaults():
    from d2slam_b200 import build, solver
    build.build()
    lib = solver.lib()
    for n in ("d2pgo_default_ceres_lm_config", "d2pgo_set_minimizer", "d2pgo_minimizer_report", "d2pgo_debug_minimizer_trace"):
        assert hasattr(lib, n) and n in pgo.PGO_EXPORTED
    got = pgo.default_ceres_lm_config()
    assert got == co.DEFAULTS


def test_minimizer_struct_layouts_match_c():
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "d2pgo.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu %d %d\\n", '
            'sizeof(d2pgo_ceres_lm_config), sizeof(d2pgo_minimizer_summary), sizeof(d2pgo_minimizer_iteration), '
            'offsetof(d2pgo_ceres_lm_config, parameter_tolerance), offsetof(d2pgo_minimizer_summary, final_cost), '
            'offsetof(d2pgo_minimizer_iteration, kind), D2PGO_MINIMIZER_CERES_LM, D2PGO_STOP_INVALID_STEPS);return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe]).decode().split()))
    assert out == [C.sizeof(pgo.CeresLmConfig), C.sizeof(pgo.MinimizerSummary), C.sizeof(pgo.MinimizerIteration),
                   pgo.CeresLmConfig.parameter_tolerance.offset, pgo.MinimizerSummary.final_cost.offset,
                   pgo.MinimizerIteration.kind.offset, pgo.MINIMIZERS["ceres_lm"], max(pgo.STOP_REASONS)]
