"""CPU oracle of the pose-graph path (TEST INFRASTRUCTURE: imported by tests/ and bench.py's cpu legs only).

numpy restatement of D2Common::RelPoseFactorAD (d2common/include/d2common/solver/RelPoseFactor.hpp:68-135) and a
Gauss-Newton solve of the same least-squares problem with scipy's sparse direct solver (pgo_lsq; the reference hands the
per-agent problems to ceres SPARSE_NORMAL_CHOLESKY + LM, d2pgo/test/d2pgo_test.cpp:95-99).  Factor level PINNED: edge_eval
is compared with the reference's own RelPoseFactorAD functor compiled into oracle/_ref/libd2ref.so (doubles for the
residual, dual numbers for its exact Jacobians; tests/test_ref_pin.py, tests/golden/ref_factors.npz); the minimiser is a
restatement (same optimum, not ceres' iterates)."""
import numpy as np

from d2slam_b200 import synth
from oracle.pgo_lsq import gauss_newton, normalize_angle


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0.0]])


def _qmul(a, b):
    return synth.quat_mul(a, b)


def edge_eval(p0, p1, rel, S):
    """RelPoseFactorAD (RelPoseFactor.hpp:76-106): r = S [q_a^-1 (p_b - p_a) - p_meas ; 2 vec(q_meas (q_a^-1 q_b)^-1)] and its exact
    tangent Jacobians (right-multiplicative retraction; the reference gets them from ceres autodiff)."""
    q0, q1, qm = p0[3:7], p1[3:7], rel[3:7]
    q0i = np.array([-q0[0], -q0[1], -q0[2], q0[3]]); q1i = np.array([-q1[0], -q1[1], -q1[2], q1[3]])
    R0i = synth.R_from_quat(q0i)
    pab = R0i @ (p1[:3] - p0[:3])
    X = _qmul(q1i, q0)
    dq = _qmul(qm, X)
    r = S @ np.concatenate([pab - rel[:3], 2.0 * dq[:3]])
    A0 = np.zeros((6, 6)); A1 = np.zeros((6, 6))
    A0[:3, :3] = -R0i; A0[:3, 3:] = _skew(pab); A1[:3, :3] = R0i
    A0[3:, 3:] = dq[3] * np.eye(3) + _skew(dq[:3])
    A1[3:, 3:] = -((qm[3] * np.eye(3) + _skew(qm[:3])) @ (X[3] * np.eye(3) - _skew(X[:3])) - np.outer(qm[:3], X[:3]))
    return r, S @ A0, S @ A1


def edge_eval_4d(pa, pb, rel_pos, rel_yaw, S):
    """RelPoseFactor4D (RelPoseFactor.hpp:216-227 + Utility::poseError4D utils.hpp:266-280), the reference's default PGO factor
    (pgo_pose_dof = PGO_POSE_4D): poses [x y z yaw]; r = S [p_meas - Rz(-yaw_a)(p_b - p_a) ; N(yaw_meas - N(yaw_b - yaw_a))] and its
    Jacobians w.r.t. the two 4-vectors (the yaw manifold's tangent is the angle itself)."""
    c, s_ = np.cos(-pa[3]), np.sin(-pa[3])
    Rz = np.array([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]]); dRz = np.array([[-s_, -c, 0.0], [c, -s_, 0.0], [0.0, 0.0, 0.0]])   # d Rz(t)/dt at t = -yaw_a
    v = pb[:3] - pa[:3]
    raw = np.concatenate([rel_pos - Rz @ v, [normalize_angle(rel_yaw - normalize_angle(pb[3] - pa[3]))]])
    A0 = np.zeros((4, 4)); A1 = np.zeros((4, 4))
    A0[:3, :3] = Rz; A0[:3, 3] = dRz @ v; A0[3, 3] = 1.0
    A1[:3, :3] = -Rz; A1[3, 3] = -1.0
    return S @ raw, S @ A0, S @ A1


def _vqmul(a, b):
    ax, ay, az, aw = a[:, 0], a[:, 1], a[:, 2], a[:, 3]; bx, by, bz, bw = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=1)


def _vskew(v):
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def _vrot(q):
    """rotation matrices of unit quaternions (x y z w), batched"""
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], 1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], 1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1)], 1)


def edges_eval(poses, ea, eb, rel, S):
    """edge_eval for all edges at once (same formulas, numpy-batched): r [E,6], J0 [E,6,6], J1 [E,6,6]."""
    p0, p1 = poses[ea], poses[eb]
    conj = np.array([-1.0, -1.0, -1.0, 1.0])
    q0i, q1i, qm = p0[:, 3:7] * conj, p1[:, 3:7] * conj, rel[:, 3:7]
    R0i = _vrot(q0i)
    pab = np.einsum("eij,ej->ei", R0i, p1[:, :3] - p0[:, :3])
    X = _vqmul(q1i, p0[:, 3:7]); dq = _vqmul(qm, X)
    raw = np.concatenate([pab - rel[:, :3], 2.0 * dq[:, :3]], axis=1)
    r = np.einsum("eij,ej->ei", S, raw)
    E = len(ea); I3 = np.eye(3)[None]
    A0 = np.zeros((E, 6, 6)); A1 = np.zeros((E, 6, 6))
    A0[:, :3, :3] = -R0i; A0[:, :3, 3:] = _vskew(pab); A1[:, :3, :3] = R0i
    A0[:, 3:, 3:] = dq[:, 3, None, None] * I3 + _vskew(dq[:, :3])
    Lm = qm[:, 3, None, None] * I3 + _vskew(qm[:, :3]); Rx = X[:, 3, None, None] * I3 - _vskew(X[:, :3])
    A1[:, 3:, 3:] = -(np.einsum("eij,ejk->eik", Lm, Rx) - np.einsum("ei,ej->eij", qm[:, :3], X[:, :3]))
    return r, np.einsum("eij,ejk->eik", S, A0), np.einsum("eij,ejk->eik", S, A1)


def solve(poses, fixed, ea, eb, rel, sqrt_info, iters=30, ftol=1e-12):
    """Gauss-Newton with a sparse direct solve (pgo_lsq.gauss_newton); returns (poses, costs)."""
    ea = np.asarray(ea); eb = np.asarray(eb); rel = np.asarray(rel, float); S = np.asarray(sqrt_info).reshape(-1, 6, 6)

    def blocks(x):
        r, J0, J1 = edges_eval(x, ea, eb, rel, S)                        # == edge_eval per edge (tests/test_pgo.py)
        return [(r, [(ea, J0), (eb, J1)])]
    return gauss_newton(poses, fixed, blocks, iters, ftol)
