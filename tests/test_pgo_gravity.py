"""Gravity prior on the 6-DoF pose graph (d2pgo's enable_gravity_prior; include/d2pgo.h d2pgo_add_gravity_priors).

CPU: the oracle (oracle/pgo_gravity_oracle.py) against the reference's own GravityPriorPerturbAD, live and through the frozen
outputs of tests/golden/ref_gravity.npz; the reference's RelPoseFactorPerturbAD at zero perturbation against pgo_oracle's
edge_eval (the factor the node runs in its 6-DoF configuration is the one the device solves); the oracle Jacobian against
finite differences; the oracle's solve.  GPU: device prior records, the converged solve against the sparse-direct oracle,
reproducibility, refusals, clearing, and the two-rank solve."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from d2slam_b200 import pgo, synth
from oracle import pgo_gravity_oracle as go
from oracle import pgo_oracle as po
from oracle import ref_gravity as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_gravity.npz")
LIVE = pytest.mark.skipif(not ref.available(), reason="reference gravity library not built")
N_CASES = 50


def close(a, b, tol):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() / max(1.0, np.abs(b).max())
    assert err <= tol, err


def tilted_quat(rng, max_tilt):
    """Random yaw, then a tilt of up to max_tilt about a random horizontal axis."""
    yaw = rng.uniform(-np.pi, np.pi); ang = rng.uniform(0.0, max_tilt); phi = rng.uniform(0.0, 2 * np.pi)
    tilt = pgo._qexp(ang * np.array([np.cos(phi), np.sin(phi), 0.0]))
    q = pgo._qmul(pgo._qyaw(yaw), tilt)
    return q / np.linalg.norm(q)


def reference_cases(n=N_CASES, seed=0):
    """Seeded inputs: pose attitude q0 and ego pose with tilts up to 80 degrees, full non-symmetric S, a perturbation theta with
    |theta| in [1e-2, 0.5], and a relative-pose edge for RelPoseFactorPerturbAD."""
    rng = np.random.default_rng(seed)
    out = {k: [] for k in ("q0", "p0", "ego", "S", "theta", "pb", "rel", "S6")}
    for _ in range(n):
        q0 = tilted_quat(rng, np.deg2rad(80)); qe = tilted_quat(rng, np.deg2rad(80))
        out["q0"].append(q0); out["p0"].append(rng.normal(0, 5, 3))
        out["ego"].append(np.concatenate([rng.normal(0, 5, 3), qe * rng.uniform(0.5, 2.0)]))   # unnormalised: Swarm::Pose normalises
        out["S"].append(10.0 * np.eye(3) + 3.0 * rng.normal(size=(3, 3)))
        th = rng.normal(size=3); out["theta"].append(th / np.linalg.norm(th) * rng.uniform(1e-2, 0.5))
        out["pb"].append(np.concatenate([rng.normal(0, 5, 3), tilted_quat(rng, np.deg2rad(80))]))
        rel = np.concatenate([rng.normal(0, 2, 3), rng.normal(size=4)]); rel[3:] /= np.linalg.norm(rel[3:])
        out["rel"].append(rel); out["S6"].append(20.0 * np.eye(6) + 5.0 * rng.normal(size=(6, 6)))
    return {k: np.array(v) for k, v in out.items()}


def reference_outputs(cases):
    """The reference functors on reference_cases (what tests/golden/make_ref_gravity_golden.py freezes)."""
    n = len(cases["q0"])
    out = {k: [] for k in ("r0", "J0", "rt", "rel_r", "rel_Ja", "rel_Jb")}
    for i in range(n):
        r, J = ref.gravity_prior_eval(cases["ego"][i], cases["S"][i], cases["q0"][i], np.concatenate([cases["p0"][i], np.zeros(3)]))
        out["r0"].append(r); out["J0"].append(J)
        out["rt"].append(ref.gravity_prior_eval(cases["ego"][i], cases["S"][i], cases["q0"][i], np.concatenate([cases["p0"][i], cases["theta"][i]]))[0])
        pb = cases["pb"][i]
        r, Ja, Jb = ref.relpose_perturb_eval(cases["rel"][i], cases["S6"][i], cases["q0"][i], pb[3:], np.concatenate([cases["p0"][i], np.zeros(3)]),
                                             np.concatenate([pb[:3], np.zeros(3)]))
        out["rel_r"].append(r); out["rel_Ja"].append(Ja); out["rel_Jb"].append(Jb)
    return {k: np.array(v) for k, v in out.items()}


def check_against_oracle(cases, outs):
    u_ego = go.ego_gravity(cases["ego"])
    for i in range(len(cases["q0"])):
        r, J = go.gravity_eval(cases["q0"][i], u_ego[i], cases["S"][i])
        close(outs["r0"][i], r, 1e-13)
        close(outs["J0"][i][:, 3:], J[:, 3:], 1e-13)
        assert np.all(outs["J0"][i][:, :3] == 0.0)                          # position columns exactly zero
        assert np.all(J[:, :3] == 0.0)
        qt = pgo._qmul(cases["q0"][i], pgo._qexp(cases["theta"][i]))         # |theta| >= 1e-2: the reference's exact chart
        close(outs["rt"][i], go.gravity_eval(qt, u_ego[i], cases["S"][i])[0], 1e-13)
        pa = np.concatenate([cases["p0"][i], cases["q0"][i]])
        r, A, B = po.edge_eval(pa, cases["pb"][i], cases["rel"][i], cases["S6"][i])
        close(outs["rel_r"][i], r, 1e-13); close(outs["rel_Ja"][i], A, 1e-13); close(outs["rel_Jb"][i], B, 1e-13)


# ----------------------------------------------------------------------------------------------- CPU
@LIVE
def test_oracle_matches_the_reference_functors_live():
    cases = reference_cases()
    check_against_oracle(cases, reference_outputs(cases))


def test_oracle_matches_the_frozen_reference_outputs():
    g = np.load(GOLD)
    cases = {k: g[f"case_{k}"] for k in reference_cases(1)}
    for k, v in reference_cases().items():
        assert np.array_equal(cases[k], v), k                                 # the golden file holds these very cases
    check_against_oracle(cases, {k: g[k] for k in ("r0", "J0", "rt", "rel_r", "rel_Ja", "rel_Jb")})


def test_cases_cover_large_tilts_and_the_exact_chart():
    c = reference_cases()
    tilt = lambda q: np.degrees(go.tilt_errors(np.concatenate([np.zeros((len(q), 3)), q], 1), np.tile([0, 0, 0, 0, 0, 0, 1.0], (len(q), 1))))
    assert tilt(c["q0"]).max() > 70 and tilt(c["q0"]).max() <= 80
    th = np.linalg.norm(c["theta"], axis=1)
    assert th.min() >= 1e-2 and th.max() <= 0.5
    assert min(np.abs(S - S.T).max() for S in c["S"]) > 0.1                  # non-symmetric S


def test_oracle_jacobian_matches_finite_differences():
    c = reference_cases(10, seed=4)
    u_ego = go.ego_gravity(c["ego"])
    h = 1e-6
    for i in range(10):
        x = np.concatenate([c["p0"][i], c["q0"][i]])
        r, J = go.gravity_eval(x[3:], u_ego[i], c["S"][i])
        Jfd = np.zeros((3, 6))
        for k in range(6):
            d = np.zeros(6); d[k] = h
            rp = go.gravity_eval(synth.pose_plus(x, d)[3:], u_ego[i], c["S"][i])[0]
            rm = go.gravity_eval(synth.pose_plus(x, -d)[3:], u_ego[i], c["S"][i])[0]
            Jfd[:, k] = (rp - rm) / (2 * h)
        close(J, Jfd, 1e-8)
        assert np.linalg.matrix_rank(J, tol=1e-9 * np.abs(J).max()) == 2      # yaw about gravity stays free


def test_batched_priors_equal_the_per_prior_function():
    c = reference_cases(20, seed=2)
    u_ego = go.ego_gravity(c["ego"])
    r, J = go.gravity_eval_batch(c["q0"], u_ego, c["S"])
    for i in range(20):
        r1, J1 = go.gravity_eval(c["q0"][i], u_ego[i], c["S"][i])
        assert np.array_equal(r[i], r1) and np.array_equal(J[i], J1)


def gravity_graph(seed=3, loops=40, full_info=False):
    g = pgo.make_pose_graph(seed=seed, n_agents=3, poses_per_agent=60, loops=loops)
    c = pgo.make_gravity_case(g, seed=seed)
    N = len(g["ids"])
    S = np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (N, 1, 1))
    if full_info:
        S = S + 2.0 * np.random.default_rng(seed).normal(size=S.shape)
    return g, c, S


def test_oracle_gravity_solve_reaches_a_stationary_point_and_corrects_roll_pitch():
    g, c, S = gravity_graph()
    idx = np.arange(len(g["ids"])); u_ego = go.ego_gravity(c["ego"])
    x, costs = go.solve_gravity(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S, iters=40, ftol=1e-14)
    g0 = go.gradient(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)
    g1 = go.gradient(x, g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)
    assert np.abs(g1).max() <= 1e-8 * np.abs(g0).max(), (np.abs(g1).max(), np.abs(g0).max())
    assert costs[-1] < costs[0]
    x0, _ = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=40, ftol=1e-14)
    rms = lambda y: float(np.sqrt(np.mean(go.tilt_errors(y, g["gt"]) ** 2)))
    assert rms(x) < 0.5 * rms(x0), (rms(x), rms(x0))                         # the priors correct the roll / pitch drift
    assert rms(g["init"]) > np.deg2rad(3.0)                                   # ... which the odometry does have


def test_make_gravity_case_keeps_chain_yaw_and_true_gravity():
    g = pgo.make_pose_graph(seed=5, n_agents=2, poses_per_agent=40, loops=20)
    c = pgo.make_gravity_case(g, sigma_tilt=0.0, seed=1)
    chain, _ = pgo._odometry_chain(g)
    assert np.array_equal(c["ego"][:, :3], chain[:, :3])
    assert np.abs(pgo.normalize_angle(pgo.quat_yaw(c["ego"][:, 3:7]) - pgo.quat_yaw(chain[:, 3:7]))).max() <= 1e-12
    assert go.tilt_errors(c["ego"], g["gt"]).max() <= 1e-7
    c = pgo.make_gravity_case(g, seed=1)
    e = go.tilt_errors(c["ego"], g["gt"])
    assert 0.2 < np.degrees(np.sqrt(np.mean(e ** 2))) < 1.5


# ----------------------------------------------------------------------------------------------- GPU
def solver(g, c=None, S=None, idx=None, fixed=None, **kw):
    s = pgo.PgoSolver(**kw)
    s.set_poses(g["ids"], g["init"], g["fixed"] if fixed is None else fixed)
    s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    if c is not None:
        idx = np.arange(len(g["ids"])) if idx is None else idx
        s.add_gravity_priors(g["ids"][idx], c["ego"][idx], None if S is None else S[idx])
    return s


@pytest.mark.gpu
def test_device_prior_records_match_the_reference_and_the_oracle():
    g = np.load(GOLD)
    cases = {k: g[f"case_{k}"] for k in reference_cases(1)}
    n = len(cases["q0"])
    ids = np.arange(n, dtype=np.int64) * 7 + 3
    poses = np.concatenate([cases["p0"], cases["q0"]], axis=1)
    s = pgo.PgoSolver()
    s.set_poses(ids, poses)
    s.add_gravity_priors(ids, cases["ego"], cases["S"])
    dev = s.debug_gravity_priors()
    assert dev.shape == (n, 21)
    r, J = go.gravity_eval_batch(cases["q0"], go.ego_gravity(cases["ego"]), cases["S"])
    for i in range(n):
        close(dev[i, :3], g["r0"][i], 1e-11); close(dev[i, 3:].reshape(3, 6), g["J0"][i], 1e-11)
        close(dev[i, :3], r[i], 1e-11); close(dev[i, 3:].reshape(3, 6), J[i], 1e-11)
        assert np.all(dev[i, 3:].reshape(3, 6)[:, :3] == 0.0)


KW_EXACT = dict(max_iterations=40, pcg_max_iterations=400, pcg_tolerance=1e-12, lambda0=0.0, function_tolerance=1e-14)


@pytest.mark.gpu
def test_converged_device_solve_matches_the_sparse_direct_oracle():
    g, c, S = gravity_graph(seed=4, loops=60, full_info=True)
    fixed = g["fixed"].copy(); fixed[70] = 1                                  # a second fixed pose; both fixed poses carry a prior
    s = solver(g, c, S, fixed=fixed, **KW_EXACT)
    rep = s.solve()
    x = s.get_poses(g["ids"])
    idx = np.arange(len(g["ids"])); u_ego = go.ego_gravity(c["ego"])
    x_ref, costs = go.solve_gravity(g["init"], fixed, g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S, iters=40, ftol=1e-14)
    assert abs(rep.initial_cost - go.cost_gravity(g["init"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)) <= 1e-10 * rep.initial_cost
    assert rep.final_cost < rep.initial_cost and abs(rep.final_cost - costs[-1]) <= 1e-8 * costs[-1], (rep.final_cost, costs[-1])
    dp, dr = synth.pose_errors(x, x_ref)
    assert dp <= 1e-6 and dr <= 1e-6, (dp, dr)
    f = fixed != 0
    assert np.array_equal(x[f], g["init"][f])


@pytest.mark.gpu
def test_gravity_solve_is_bitwise_reproducible():
    g, c, S = gravity_graph(seed=6, full_info=True)
    xs = []
    for _ in range(2):
        s = solver(g, c, S, max_iterations=20, pcg_max_iterations=200, pcg_tolerance=1e-6, lambda0=1e-4)
        r = s.solve(); xs.append((s.get_poses(g["ids"]), r.final_cost, r.iterations, r.pcg_iterations)); s.close()
    assert np.array_equal(xs[0][0], xs[1][0]) and xs[0][1:] == xs[1][1:]


def raw_add(s, n, ids, ego, S):
    from d2slam_b200.solver import lib
    p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    return lib().d2pgo_add_gravity_priors(s.h, C.c_int32(n), p(ids), p(ego), p(S))


def solved(s, g):
    r = s.solve()
    return s.get_poses(g["ids"]), r.final_cost, r.iterations, r.pcg_iterations


KW_INEXACT = dict(max_iterations=15, pcg_max_iterations=200, pcg_tolerance=1e-6, lambda0=1e-4)


@pytest.mark.gpu
def test_bad_gravity_priors_are_refused_and_leave_the_handle_unchanged():
    g, c, S = gravity_graph(seed=7)
    ids, ego = g["ids"], c["ego"]
    s = solver(g, **KW_INEXACT)
    I = np.tile(np.eye(3), (3, 1, 1))
    with pytest.raises(RuntimeError, match="rc=2.*unknown pose id"):
        s.add_gravity_priors(np.array([ids[0], 999_999_999]), ego[:2])
    with pytest.raises(RuntimeError, match="rc=2.*already has a gravity prior"):
        s.add_gravity_priors(np.array([ids[1], ids[2], ids[1]]), ego[:3])
    bad = ego[:3].copy(); bad[1, 0] = np.nan
    with pytest.raises(RuntimeError, match="rc=2.*non-finite"):
        s.add_gravity_priors(ids[:3], bad)
    bS = I.copy(); bS[2, 1, 1] = np.inf
    with pytest.raises(RuntimeError, match="rc=2.*non-finite"):
        s.add_gravity_priors(ids[:3], ego[:3], bS)
    bad = ego[:3].copy(); bad[2, 3:7] = 0.0
    with pytest.raises(RuntimeError, match="rc=2.*zero ego quaternion"):
        s.add_gravity_priors(ids[:3], bad)
    assert raw_add(s, -1, ids[:1], ego[:1], I[:1]) == 1
    assert raw_add(s, 2, ids[:2], None, I[:2]) == 1
    assert s.n_priors == 0 and s.debug_gravity_priors().shape == (0, 21)
    # nothing of a refused call was kept: the handle solves as one that never saw the calls
    ref = solver(g, **KW_INEXACT)
    a, b = solved(s, g), solved(ref, g)
    assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
    # a second prior on a pose that already has one, across calls
    s.add_gravity_priors(ids[:2], ego[:2])
    with pytest.raises(RuntimeError, match="rc=2.*already has a gravity prior"):
        s.add_gravity_priors(ids[1:3], ego[1:3])
    # 4-DoF handles refuse the prior (d2pgo skips it for 4-DoF)
    h = pgo.pose_graph_to_4d(g)
    s4 = pgo.PgoSolver(pose_dof=4)
    s4.set_poses_4d(h["ids"], h["init"], h["fixed"])
    with pytest.raises(RuntimeError, match="rc=5.*pose_dof = 4"):
        s4.add_gravity_priors(ids[:2], ego[:2])
    with pytest.raises(RuntimeError, match="rc=5"):
        s4.debug_gravity_priors()
    assert raw_add(s4, 1, ids[:1], ego[:1], I[:1]) == 5


@pytest.mark.gpu
def test_set_poses_clears_the_priors_and_an_empty_call_changes_nothing():
    g, c, S = gravity_graph(seed=8, full_info=True)
    ref = solved(solver(g, **KW_INEXACT), g)
    # set_poses removes the priors (and the edges): reload the same graph without priors
    s = solver(g, c, S, **KW_INEXACT)
    with_priors = solved(s, g)
    assert with_priors[1] != ref[1]
    s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    assert s.debug_gravity_priors().shape == (0, 21)
    a = solved(s, g)
    assert np.array_equal(a[0], ref[0]) and a[1:] == ref[1:]
    # an n = 0 call changes nothing
    s2 = solver(g, **KW_INEXACT)
    assert raw_add(s2, 0, None, None, None) == 0
    s2.add_gravity_priors(np.zeros(0, np.int64), np.zeros((0, 7)))
    b = solved(s2, g)
    assert np.array_equal(b[0], ref[0]) and b[1:] == ref[1:]


@pytest.mark.gpu
def test_device_priors_correct_roll_and_pitch():
    g, c, S = gravity_graph(seed=3)
    x0 = solver(g, **KW_EXACT); x0.solve(); x0 = x0.get_poses(g["ids"])
    x1 = solver(g, c, **KW_EXACT); x1.solve(); x1 = x1.get_poses(g["ids"])
    rms = lambda y: float(np.sqrt(np.mean(go.tilt_errors(y, g["gt"]) ** 2)))
    assert rms(x1) < 0.5 * rms(x0), (rms(x1), rms(x0))


@pytest.mark.gpu
def test_two_rank_gravity_pose_graph_matches_single_rank():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", os.path.join(ROOT, "tools", "pgo_multi_gpu_check.py"), "--gravity"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-2000:]); sys.stderr.write(out.stderr[-2000:])
    assert out.returncode == 0 and "PGO_MULTI_GPU_CHECK PASS" in out.stdout
