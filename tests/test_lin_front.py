"""The linearisation front (k_misc_lin: Hcc reset, prior, ADMM terms; k_imu_lin: IMU factors) on batches that mix
window shapes in one launch, against the CPU oracle."""
import numpy as np
import pytest

from d2slam_b200 import abi, synth
from helpers import relerr, state_diff, state_of

pytestmark = pytest.mark.gpu


def load(pr, solver, window=None, sb_const=None):
    """synth.Problem.load with an optional constness mask on the speed-bias blocks."""
    args = () if window is None else (window,)
    solver.set_blocks(*args, abi.POSE, pr["frame_ids"], pr["poses"], pr["pose_const"])
    solver.set_blocks(*args, abi.EXTRINSIC, pr["cam_ids"], pr["ext"], pr["ext_const"])
    solver.set_blocks(*args, abi.SPEED_BIAS, pr["sb_ids"], pr["sb"], sb_const)
    solver.set_blocks(*args, abi.TD, np.zeros(1, np.int64), np.array([pr["td"]]), np.array([pr["td_const"]], np.uint8))
    solver.set_blocks(*args, abi.LANDMARK, pr["lm_ids"], pr["inv_dep"], None)
    solver.add_proj(*args, pr["obs"])
    if len(pr["imu"]):
        solver.add_imu(*args, pr["imu"])
    if pr.get("prior") is not None:
        A, b, refs, x0 = pr["prior"]
        solver.set_prior_info(*args, A, b, refs, x0)
    if pr.get("consensus") is not None:
        refs, slots, n_slots = pr["consensus"]
        solver.set_consensus(*args, refs, slots, n_slots)


def mixed_batch():
    """(problem, speed-bias constness mask) per window: a long IMU chain, a window whose IMU list is empty, a window with
    constant pose and speed-bias blocks (IMU columns -1 on either end), and a stereo window with a prior."""
    long_chain = synth.make_window(seed=61, n_frames=40, n_landmarks=150)
    assert len(long_chain["imu"]) == 39
    no_imu = synth.make_window(seed=62, n_landmarks=80)
    no_imu["imu"] = no_imu["imu"][:0]
    const = synth.make_window(seed=63, n_landmarks=80, with_prior=False)
    pc = np.asarray(const["pose_const"], np.uint8).copy()
    pc[[0, 3]] = 1
    const["pose_const"] = pc
    sbc = np.zeros(len(const["sb_ids"]), np.uint8)
    sbc[[1, 4]] = 1
    stereo = synth.make_window(seed=64, cams="stereo", n_landmarks=80)
    return [(long_chain, None), (no_imu, None), (const, sbc), (stereo, None)]


def test_mixed_batch_normal_equations():
    from d2slam_b200.solver import Solver
    from oracle import orc
    batch = mixed_batch()
    s = Solver(max_windows=len(batch))
    for i, (pr, sbc) in enumerate(batch):
        load(pr, s, i, sbc)
    s.finalize()
    s.debug_linearize()
    for i, (pr, sbc) in enumerate(batch):
        o = orc.Oracle()
        load(pr, o, None, sbc)
        o.debug_linearize()
        for item in (abi.DBG_COST, abi.DBG_HCC, abi.DBG_GC):
            assert relerr(s.debug_get(i, item), o.debug_get(item)) <= 1e-10, (i, item)
    # the IMU factors alone, through the device path the linearisation runs
    a = s.debug_get(0, abi.DBG_IMU_RESJAC).reshape(-1, 465)
    assert a.shape[0] == 39 and np.isfinite(a).all()
    assert s.debug_get(1, abi.DBG_IMU_RESJAC).size == 0


def test_mixed_batch_admm_fixed_schedule():
    """ADMM windows go through the same kernels: a 4-agent swarm in one handle, one agent without IMU factors and one
    with constant speed-bias blocks, against the oracle's in-process ADMM."""
    from d2slam_b200.solver import Solver
    from oracle import orc
    sw = synth.make_swarm(seed=83, n_agents=4, n_landmarks=120, shared_per_pair=20)
    sw[1]["imu"] = sw[1]["imu"][:0]
    masks = [None, None, np.zeros(len(sw[2]["sb_ids"]), np.uint8), None]
    masks[2][[2, 5]] = 1
    steps, iters = 2, 4
    cfg = dict(consensus_max_steps=steps, max_num_iterations=iters)
    ags = []
    for p, m in zip(sw, masks):
        a = orc.Oracle(**cfg)
        load(p, a, None, m)
        ags.append(a)
    ro = orc.admm_solve(ags, fixed_mode=True)
    s = Solver(max_windows=len(sw), **cfg)
    for i, (p, m) in enumerate(zip(sw, masks)):
        load(p, s, i, m)
    s.finalize()
    rs = s.solve_fixed(iters)
    for i, p in enumerate(sw):
        assert rs[i].total_iterations == ro[i].total_iterations
        assert abs(rs[i].final_cost - ro[i].final_cost) <= 1e-6 * max(1.0, ro[i].final_cost), (i, rs[i].final_cost, ro[i].final_cost)
        d = state_diff(state_of(s, p, i), state_of(ags[i], p))
        assert d["pos"] <= 1e-6 and d["rot"] <= 1e-6 and d["lm_rel"] <= 1e-5, (i, d)
