"""4-DoF pose graph (d2pgo's default configuration: RelPoseFactor4D on [x y z yaw] poses, include/d2pgo.h pose_dof = 4):
the batched oracle against the per-edge factor and the frozen reference outputs, the oracle's solve, edge sharding, the 7 <-> 4
pose conversions; on the GPU the device edge records against the reference functor's outputs and the oracle, the converged
solution across yaw +-pi against the sparse-direct oracle, reproducibility, the ABI's refusals, and the multi-rank solve."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pgo4d_oracle as p4
from oracle import pgo_oracle as po

import test_ref_pin as trp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_factors.npz")


def graph_4d(seed=1, n_agents=3, n=40, loops=120, full_info=False):
    h = pgo.pose_graph_to_4d(pgo.make_pose_graph(seed=seed, n_agents=n_agents, poses_per_agent=n, loops=loops), seed=seed + 100)
    S = h["sqrt_info"].reshape(-1, 4, 4)
    if full_info:
        S = S + 0.5 * np.random.default_rng(seed).normal(size=S.shape)      # full square-root information
    return h, S


def rotate_about_z(g, theta):
    """The graph's ground truth turned by theta about the world z axis (distances, so the loop closures, unchanged)."""
    c, s = np.cos(theta), np.sin(theta)
    gt = g["gt"].copy()
    gt[:, 0], gt[:, 1] = c * g["gt"][:, 0] - s * g["gt"][:, 1], s * g["gt"][:, 0] + c * g["gt"][:, 1]
    gt[:, 3:7] = pgo._qmul(np.array([0.0, 0.0, np.sin(theta / 2), np.cos(theta / 2)]), g["gt"][:, 3:7])
    return dict(g, gt=gt)


def wrapped_graph():
    """4 agents; ground truth turned so that agent 1's trajectory crosses yaw +-pi."""
    g = pgo.make_pose_graph(seed=6, n_agents=4, poses_per_agent=60, loops=300)
    yaw1 = pgo.poses_to_4d(g["gt"][g["agent"] == 1])[:, 3]
    h = pgo.pose_graph_to_4d(rotate_about_z(g, np.pi - np.median(yaw1)), seed=6)
    y = h["gt"][h["agent"] == 1, 3]
    assert y.max() > 2.8 and y.min() < -2.8          # the trajectory does cross +-pi
    return h


def position_yaw_errors(x, y):
    return np.linalg.norm(x[:, :3] - y[:, :3], axis=1).max(), np.abs(pgo.normalize_angle(x[:, 3] - y[:, 3])).max()


# ----------------------------------------------------------------------------------------------- CPU
def test_batched_4d_linearisation_equals_the_per_edge_function():
    h, S = graph_4d(seed=7, full_info=True)
    r, J0, J1 = p4.edges_eval_4d(h["init"], h["ea"], h["eb"], h["rel"], S)
    for e in range(len(h["ea"])):
        r1, a, b = po.edge_eval_4d(h["init"][h["ea"][e]], h["init"][h["eb"][e]], h["rel"][e, :3], h["rel"][e, 3], S[e])
        assert np.abs(r[e] - r1).max() <= 1e-12 * max(1.0, np.abs(r1).max())
        assert np.abs(J0[e] - a).max() <= 1e-12 * np.abs(a).max() and np.abs(J1[e] - b).max() <= 1e-12 * np.abs(b).max()


def relpose4d_inputs():
    """relpose4d_cases() of test_ref_pin as 4-DoF inputs: measurement yaw taken from `rel` as check_relpose4d takes it."""
    cases = trp.relpose4d_cases()
    poses = np.array([p for c in cases for p in (c["pa"], c["pb"])])
    rel = np.array([np.concatenate([c["rel"][:3], [pgo.quat_yaw(c["rel"][3:7])]]) for c in cases])
    S = np.array([c["S"] for c in cases])
    ea = np.arange(0, 2 * len(cases), 2); eb = ea + 1
    return poses, ea, eb, rel, S


def test_batched_4d_linearisation_matches_the_golden_reference_vectors():
    """edges_eval_4d on the reference-pinned cases (yaw wrap included) against RelPoseFactor4D's frozen outputs."""
    g = np.load(GOLD)
    poses, ea, eb, rel, S = relpose4d_inputs()
    r, J0, J1 = p4.edges_eval_4d(poses, ea, eb, rel, S)
    for i in range(len(ea)):
        trp.close(r[i], g[f"relpose4d{i}_r"], 1e-13); trp.close(J0[i], g[f"relpose4d{i}_Ja"], 1e-13); trp.close(J1[i], g[f"relpose4d{i}_Jb"], 1e-13)


def test_oracle_4d_solve_lowers_the_cost_and_approaches_ground_truth():
    h = wrapped_graph()
    x, costs = p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"])
    assert costs[-1] < 0.1 * costs[0]
    e0, _ = position_yaw_errors(h["init"], h["gt"]); e1, _ = position_yaw_errors(x, h["gt"])
    assert e1 < 0.5 * e0, (e0, e1)
    assert np.all(x[:, 3] >= -np.pi) and np.all(x[:, 3] < np.pi)
    assert np.array_equal(x[0], h["init"][0])


def test_4d_edge_sharding_sums_to_the_full_normal_equations():
    """What the multi-GPU path relies on for D = 4: J^T J p summed over edge shards (e % 3) == the full product."""
    h, S = graph_4d(seed=4, full_info=True)
    N = len(h["ids"]); p = np.random.default_rng(0).normal(size=(N, 4))
    _, J0, J1 = p4.edges_eval_4d(h["init"], h["ea"], h["eb"], h["rel"], S)

    def product(sel):
        y = np.zeros((N, 4))
        for e in sel:
            a, b = h["ea"][e], h["eb"][e]
            t = J0[e] @ p[a] + J1[e] @ p[b]; y[a] += J0[e].T @ t; y[b] += J1[e].T @ t
        return y
    E = len(h["ea"]); full = product(range(E))
    parts = sum(product(range(r, E, 3)) for r in range(3))
    assert np.abs(full - parts).max() <= 1e-9 * np.abs(full).max()


def test_poses_from_4d_inverts_poses_to_4d():
    g = pgo.make_pose_graph(seed=3, n_agents=2, poses_per_agent=50, loops=20)
    p = g["gt"]
    assert np.abs(pgo.poses_from_4d(pgo.poses_to_4d(p), p) - p).max() <= 1e-14
    # a solved yaw replaces the ego yaw and keeps the ego pose's roll and pitch
    x4 = pgo.poses_to_4d(p); x4[:, 3] += 0.3
    q = pgo.poses_from_4d(x4, p)
    assert np.abs(pgo.normalize_angle(pgo.quat_yaw(q[:, 3:7]) - x4[:, 3])).max() <= 1e-12
    tilt = lambda qq: pgo._qmul(pgo._qconj(pgo._qyaw(pgo.quat_yaw(qq))), qq)
    assert np.abs(tilt(q[:, 3:7]) - tilt(p[:, 3:7])).max() <= 1e-12


def test_pose_graph_to_4d_keeps_the_graph():
    g = pgo.make_pose_graph(seed=2, n_agents=3, poses_per_agent=30, loops=60)
    h = pgo.pose_graph_to_4d(g, seed=5)
    assert np.array_equal(h["ea"], g["ea"]) and np.array_equal(h["id_b"], g["id_b"]) and h["sqrt_info"].shape == (len(g["ea"]), 16)
    assert np.array_equal(h["init"][0], h["gt"][0]) and h["fixed"][0] == 1 and h["fixed"][1:].sum() == 0
    # noise-free measurements would give zero residual at the ground truth: the noise is what is left
    r = p4.edges_eval_4d(h["gt"], h["ea"], h["eb"], h["rel"], np.tile(np.eye(4), (len(h["ea"]), 1, 1)))[0]
    assert np.abs(r[:, :3]).max() < 0.5 and np.abs(r[:, 3]).max() < np.deg2rad(6.0)


def test_bad_pose_dof_is_refused_before_any_device_work():
    with pytest.raises(RuntimeError, match="pose_dof"):
        pgo.PgoSolver(pose_dof=5)


def test_pose_dof_takes_the_reserved_slot():
    """d2pgo_config keeps its size and offsets; pose_dof sits where `reserved` was."""
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "d2pgo.h"\nint main(void){printf("%zu %zu %zu\\n", sizeof(d2pgo_config), '
            'offsetof(d2pgo_config, pose_dof), offsetof(d2pgo_config, pcg_tolerance));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe]).decode().split()))
    assert out == [40, 12, 16] == [C.sizeof(pgo.PgoConfig), pgo.PgoConfig.pose_dof.offset, pgo.PgoConfig.pcg_tolerance.offset]
    cfg = pgo.PgoConfig()
    from d2slam_b200.solver import lib
    lib().d2pgo_default_config(C.byref(cfg))
    assert cfg.pose_dof == 0


# ----------------------------------------------------------------------------------------------- GPU
def solver_4d(h, S=None, **kw):
    s = pgo.PgoSolver(pose_dof=4, **kw)
    s.set_poses_4d(h["ids"], h["init"], h["fixed"])
    s.add_edges_4d(h["id_a"], h["id_b"], h["rel"], (h["sqrt_info"] if S is None else S).reshape(-1, 16))
    return s


@pytest.mark.gpu
def test_4d_edges_on_device_match_the_reference_functor():
    """Device r | J_a | J_b of RelPoseFactor4D vs the reference functor's outputs frozen in tests/golden/ref_factors.npz
    (doubles for the residual, dual numbers for the Jacobians), yaw-wrap case included."""
    g = np.load(GOLD)
    poses, ea, eb, rel, S = relpose4d_inputs()
    ids = np.arange(len(poses), dtype=np.int64)
    s = pgo.PgoSolver(pose_dof=4)
    s.set_poses_4d(ids, poses); s.add_edges_4d(ids[ea], ids[eb], rel, S.reshape(-1, 16))
    dev = s.debug_edges()
    assert dev.shape == (len(ea), 36)
    for i in range(len(ea)):
        for blk, want in ((dev[i, :4], g[f"relpose4d{i}_r"]), (dev[i, 4:20], g[f"relpose4d{i}_Ja"]), (dev[i, 20:], g[f"relpose4d{i}_Jb"])):
            want = np.ravel(want)
            assert np.abs(blk - want).max() <= 1e-11 * max(1.0, np.abs(want).max()), i


@pytest.mark.gpu
def test_4d_edges_on_device_match_the_oracle():
    h, S = graph_4d(seed=5, full_info=True)
    dev = solver_4d(h, S).debug_edges()
    r, J0, J1 = p4.edges_eval_4d(h["init"], h["ea"], h["eb"], h["rel"], S)
    ref = np.concatenate([r, J0.reshape(-1, 16), J1.reshape(-1, 16)], axis=1)
    assert dev.shape == ref.shape
    scale = np.maximum(1.0, np.abs(ref).max(axis=1))
    assert (np.abs(dev - ref).max(axis=1) <= 1e-11 * scale).all()


KW_EXACT = dict(max_iterations=40, pcg_max_iterations=400, pcg_tolerance=1e-12, lambda0=0.0, function_tolerance=1e-14)


@pytest.mark.gpu
def test_4d_converged_solution_across_yaw_pi_matches_sparse_direct_oracle():
    h = wrapped_graph()
    s = solver_4d(h, **KW_EXACT)
    rep = s.solve()
    x = s.get_poses_4d(h["ids"])
    x_ref, costs = p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"], iters=40)
    assert rep.final_cost < rep.initial_cost and abs(rep.final_cost - costs[-1]) <= 1e-8 * costs[-1], (rep.final_cost, costs[-1])
    dp, dyaw = position_yaw_errors(x, x_ref)
    assert dp <= 1e-6 and dyaw <= 1e-6, (dp, dyaw)
    assert np.all(x[:, 3] >= -np.pi) and np.all(x[:, 3] < np.pi)
    f = h["fixed"] != 0
    assert np.array_equal(x[f], h["init"][f])
    e0, _ = position_yaw_errors(h["init"], h["gt"]); e1, _ = position_yaw_errors(x, h["gt"])
    assert e1 < 0.5 * e0, (e0, e1)


@pytest.mark.gpu
def test_4d_solve_is_bitwise_reproducible():
    h = wrapped_graph()
    xs = []
    for _ in range(2):
        s = solver_4d(h, max_iterations=20, pcg_max_iterations=200, pcg_tolerance=1e-6, lambda0=1e-4)
        s.solve(); xs.append(s.get_poses_4d(h["ids"])); s.close()
    assert np.array_equal(xs[0], xs[1])


@pytest.mark.gpu
def test_mixed_6dof_and_4dof_calls_are_refused():
    h, _ = graph_4d(seed=2, n=10, loops=10)
    g = pgo.make_pose_graph(seed=2, n_agents=3, poses_per_agent=10, loops=10)
    with pytest.raises(RuntimeError, match="pose_dof"):
        pgo.PgoSolver(pose_dof=7)
    s4 = solver_4d(h)
    with pytest.raises(RuntimeError, match="pose_dof = 4"):
        s4.set_poses(g["ids"], g["init"], g["fixed"])
    with pytest.raises(RuntimeError, match="pose_dof = 4"):
        s4.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    with pytest.raises(RuntimeError, match="pose_dof = 4"):
        s4.get_poses(g["ids"])
    s6 = pgo.PgoSolver()
    s6.set_poses(g["ids"], g["init"], g["fixed"])
    with pytest.raises(RuntimeError, match="pose_dof = 6"):
        s6.set_poses_4d(h["ids"], h["init"], h["fixed"])
    with pytest.raises(RuntimeError, match="pose_dof = 6"):
        s6.add_edges_4d(h["id_a"], h["id_b"], h["rel"], h["sqrt_info"])
    with pytest.raises(RuntimeError, match="pose_dof = 6"):
        s6.get_poses_4d(h["ids"])
    # both handles still work after the refusals
    r4 = s4.solve()
    assert r4.final_cost <= r4.initial_cost
    s6.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    r6 = s6.solve()
    assert r6.final_cost <= r6.initial_cost


@pytest.mark.gpu
def test_two_rank_4d_pose_graph_matches_single_rank():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tools", "pgo_multi_gpu_check.py"), "--dof", "4"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-2000:]); sys.stderr.write(out.stderr[-2000:])
    assert out.returncode == 0 and "PGO_MULTI_GPU_CHECK PASS" in out.stdout
