"""L1 on the device against the REFERENCE's own factor classes (the unmodified D2SLAM sources compiled by oracle/Makefile.ref,
their outputs on these seeded windows frozen in tests/golden/ref_cases.npz by tests/golden/make_ref_cases_golden.py): the CUDA
path's residual and tangent Jacobian vs ProjectionTwoFrame*Factor::Evaluate and IMUFactor::Evaluate; the consensus factor
vs the oracle's ConsenusPoseFactor, which tests/test_ref_pin.py pins to the reference class."""
import os

import numpy as np
import pytest

from d2slam_b200 import abi, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cases.npz")
PROJ_CASES = [dict(seed=2, cams="stereo", estimate_extrinsic=True, estimate_td=True, td_offset=0.002, n_landmarks=60, n_frames=5),
              dict(seed=5, cams="quad", n_landmarks=80, n_frames=4)]
IMU_CASE = dict(seed=9, n_landmarks=40, n_frames=6)


def scaled(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1.0))


@pytest.mark.parametrize("case", PROJ_CASES)
def test_reprojection_factors_on_device_match_reference_classes(case):
    from d2slam_b200.solver import Solver
    g = np.load(GOLD)
    pr = synth.make_window(**case)
    case = PROJ_CASES.index(case)
    s = Solver(); pr.load(s, 0); s.finalize(); s.debug_linearize()
    dev = s.debug_get(0, abi.DBG_PROJ_RESJAC).reshape(-1, 81)
    want = g[f"proj{case}_want"]
    assert len(dev) == len(pr["obs"]) == len(want)
    worst = 0.0
    for k, w in enumerate(want):
        # device layout: r (3) | J (3 x 26): [pose_i 6 | pose_j 6 | ext_a 6 | ext_b 6 | lambda | td]
        t = int(pr["obs"]["type"][k])
        d = dev[k]; J = d[3:].reshape(3, 26)[:2]
        worst = max(worst, scaled(d[:2], w[:, 0]))
        cols = {abi.PROJ_2F1C: (0, 6, 12), abi.PROJ_2F2C: (0, 6, 12, 18), abi.PROJ_1F2C: (12, 18)}[t]
        for off in cols:
            worst = max(worst, scaled(J[:, off:off + 6], w[:, 1 + off:7 + off]))
        worst = max(worst, scaled(J[:, 24], w[:, 25]), scaled(J[:, 25], w[:, 26]))
    assert worst <= 1e-12, worst
    assert len(set(int(t) for t in pr["obs"]["type"])) >= 2


def test_imu_factors_on_device_match_reference_class():
    from d2slam_b200.solver import Solver
    g = np.load(GOLD)
    pr = synth.make_window(**IMU_CASE)
    s = Solver(); pr.load(s, 0); s.finalize(); s.debug_linearize()
    dev = s.debug_get(0, abi.DBG_IMU_RESJAC).reshape(-1, 465)
    assert len(dev) == len(pr["imu"]) == len(g["imu_r"]) > 0
    for k in range(len(dev)):
        r, Jr, si = g["imu_r"][k], g["imu_J"][k], g["imu_sqrt_info"][k]
        J = dev[k][15:].reshape(15, 30)
        # sqrt_info = LLT(cov^-1)^T of a 1e8-conditioned covariance: compare un-whitened (1e-10) and whitened (1e-7)
        U = np.linalg.inv(si)
        assert scaled(U @ dev[k][:15], U @ r) <= 1e-10 and scaled(U @ J, U @ Jr) <= 1e-10
        assert scaled(dev[k][:15], r) <= 1e-7 and scaled(J, Jr) <= 1e-7


def test_consensus_factors_on_device_match_reference_class():
    """z and tilde come out of the device's own ADMM steps, so the reference values cannot be frozen ahead of the run: the
    factor is evaluated by the oracle's restatement, which test_ref_pin holds to the reference class at 1e-14."""
    from d2slam_b200.solver import Solver
    from test_ref_pin import orc_cons
    sw = synth.make_swarm(seed=12, n_agents=3, n_landmarks=60, shared_per_pair=20, n_frames=5)
    cfg = dict(consensus_max_steps=2, max_num_iterations=4, rho_frame_T=10.0, rho_frame_theta=1000.0)
    s = Solver(max_windows=3, **cfg)
    for i, p in enumerate(sw):
        p.load(s, i)
    s.finalize(); s.solve_fixed(4)       # leaves z, tilde of the last sub-step and the solved x on the device
    n = 0
    for i in range(3):
        rec = s.debug_get(i, abi.DBG_CONS_RESJAC).reshape(-1, 62)
        for q in rec:
            if not np.any(q):
                continue
            x, z, tl, r, J = q[:7], q[7:14], q[14:20], q[20:26], q[26:].reshape(6, 6)
            rr, Jr = orc_cons(dict(z=z.copy(), x=x.copy(), tt=tl[:3].copy(), th=tl[3:].copy(), rho_T=cfg["rho_frame_T"], rho_theta=cfg["rho_frame_theta"]))
            assert scaled(r, rr) <= 1e-13 and scaled(J, Jr[:, :6]) <= 1e-13
            n += 1
    assert n >= 30
