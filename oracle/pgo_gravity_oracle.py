"""CPU oracle of the pose graph's gravity prior (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

d2pgo's enable_gravity_prior (D2PGO::setupGravityPriorFactors, d2pgo/src/d2pgo.cpp:530-559) adds one
D2Common::GravityPriorPerturbAD residual (d2common/include/d2common/solver/GravityPrior.hpp:8-46) per frame:

    u = R(q_i)^T e3   (the third row of R_i),   u_ego = R(q_ego)^T e3,   r = S^T (u - u_ego)

(the reference forms the row R_i.row(2) - R_ego.row(2) and calls applyOnTheRight(S)).  In the tangent of the
right-multiplicative pose retraction (q <- q (x) [1, dtheta / 2], p <- p + dp): dr/ddtheta = S^T [u]x, dr/ddp = 0; rank 2, yaw
about gravity stays free.  Factor level PINNED: gravity_eval is compared with the reference's own functor compiled into
oracle/_ref/libd2ref_gravity.so (tests/test_pgo_gravity.py, tests/golden/ref_gravity.npz).  solve_gravity is the sparse-direct
Gauss-Newton of pgo_oracle.solve with the priors' rows appended (same optimum as ceres, not its iterates)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from d2slam_b200 import synth
from oracle.pgo_oracle import _vrot, _vskew, edges_eval


def ego_gravity(ego7):
    """u_ego = R(q_ego)^T e3 of [x y z qx qy qz qw] ego poses (attitude normalised as Swarm::Pose stores it), [G, 3]."""
    q = np.asarray(ego7, np.float64).reshape(-1, 7)[:, 3:7]
    q = q / np.sqrt((q * q).sum(axis=1, keepdims=True))
    return _vrot(q)[:, 2, :]


def gravity_eval(q, u_ego, S):
    """One prior at attitude q [qx qy qz qw]: r (3) and the 3 x 6 tangent Jacobian [0 | S^T [u]x]."""
    r, J = gravity_eval_batch(np.asarray(q, np.float64)[None], np.asarray(u_ego, np.float64)[None], np.asarray(S, np.float64).reshape(1, 3, 3))
    return r[0], J[0]


def gravity_eval_batch(q, u_ego, S):
    """gravity_eval for G priors at once: q [G,4], u_ego [G,3], S [G,3,3] -> r [G,3], J [G,3,6]."""
    q = np.asarray(q, np.float64); S = np.asarray(S, np.float64).reshape(-1, 3, 3)
    u = _vrot(q)[:, 2, :]
    St = np.transpose(S, (0, 2, 1))
    r = np.einsum("gij,gj->gi", St, u - np.asarray(u_ego, np.float64))
    J = np.zeros((len(q), 3, 6))
    J[:, :, 3:] = np.einsum("gij,gjk->gik", St, _vskew(u))
    return r, J


def priors_eval(poses, idx, u_ego, S):
    """gravity_eval_batch at poses[idx] ([N,7] poses, idx [G] pose indices)."""
    return gravity_eval_batch(np.asarray(poses, np.float64)[np.asarray(idx)][:, 3:7], u_ego, S)


def cost_gravity(poses, ea, eb, rel, sqrt_info, idx, u_ego, S):
    """1/2 sum |r|^2 over the edges and the priors."""
    poses = np.asarray(poses, np.float64)
    re = edges_eval(poses, np.asarray(ea), np.asarray(eb), np.asarray(rel, np.float64), np.asarray(sqrt_info).reshape(-1, 6, 6))[0]
    rg = priors_eval(poses, idx, u_ego, S)[0] if len(idx) else np.zeros((0, 3))
    return 0.5 * float(np.sum(re * re) + np.sum(rg * rg))


def _system(x, col, ea, eb, rel, S6, idx, u_ego, S3):
    """Stacked residual and sparse Jacobian (free-pose tangent columns) of edges + priors."""
    nfree = int((col >= 0).sum())
    r_e, J0, J1 = edges_eval(x, ea, eb, rel, S6)
    E = len(ea); rr6, cc6 = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
    rows, cols, vals = [], [], []
    for blk, J in ((ea, J0), (eb, J1)):
        keep = col[blk] >= 0
        e_idx = np.nonzero(keep)[0]
        rows.append((6 * e_idx[:, None, None] + rr6[None]).ravel()); cols.append((col[blk[keep]][:, None, None] + cc6[None]).ravel()); vals.append(J[keep].ravel())
    G = len(idx)
    r_all = r_e.ravel()
    if G:
        r_g, Jg = priors_eval(x, idx, u_ego, S3)
        rr3, cc3 = np.meshgrid(np.arange(3), np.arange(6), indexing="ij")
        keep = col[idx] >= 0
        g_idx = np.nonzero(keep)[0]
        rows.append((6 * E + 3 * g_idx[:, None, None] + rr3[None]).ravel()); cols.append((col[idx[keep]][:, None, None] + cc3[None]).ravel()); vals.append(Jg[keep].ravel())
        r_all = np.concatenate([r_all, r_g.ravel()])
    J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * E + 3 * G, 6 * nfree))
    return r_all, J


def gradient(poses, fixed, ea, eb, rel, sqrt_info, idx, u_ego, S):
    """J^T r over the free poses' tangents, [n_free, 6]."""
    x = np.asarray(poses, np.float64); N = len(x)
    free = np.nonzero(np.asarray(fixed) == 0)[0]; col = -np.ones(N, int); col[free] = np.arange(len(free)) * 6
    r, J = _system(x, col, np.asarray(ea), np.asarray(eb), np.asarray(rel, np.float64), np.asarray(sqrt_info).reshape(-1, 6, 6),
                   np.asarray(idx, int), np.asarray(u_ego, np.float64).reshape(-1, 3), np.asarray(S, np.float64).reshape(-1, 3, 3))
    return (J.T @ r).reshape(-1, 6)


def solve_gravity(poses, fixed, ea, eb, rel, sqrt_info, idx, u_ego, S, iters=30, ftol=1e-12):
    """Gauss-Newton with a sparse direct solve over the edges (RelPoseFactorAD) and the gravity priors; returns (poses, costs).
    idx [G] pose index of each prior, u_ego [G,3] (ego_gravity), S [G,3,3]."""
    x = np.array(poses, float); N = len(x)
    free = np.nonzero(np.asarray(fixed) == 0)[0]; col = -np.ones(N, int); col[free] = np.arange(len(free)) * 6
    ea = np.asarray(ea); eb = np.asarray(eb); rel = np.asarray(rel, float); S6 = np.asarray(sqrt_info).reshape(-1, 6, 6)
    idx = np.asarray(idx, int); u_ego = np.asarray(u_ego, float).reshape(-1, 3); S3 = np.asarray(S, float).reshape(-1, 3, 3)
    costs = []
    for it in range(iters):
        r_all, J = _system(x, col, ea, eb, rel, S6, idx, u_ego, S3)
        c = 0.5 * float(r_all @ r_all); costs.append(c)
        if it and abs(costs[-2] - c) <= ftol * max(c, 1e-300):
            break
        H = (J.T @ J).tocsc(); g = J.T @ r_all
        dx = spla.spsolve(H + 1e-12 * sp.identity(H.shape[0], format="csc"), -g)
        for i in free:
            x[i] = synth.pose_plus(x[i], dx[col[i]:col[i] + 6])
    return x, costs


def tilt_errors(poses, gt):
    """Roll / pitch error per pose: the angle between the gravity directions R^T e3 of the two attitudes [rad]."""
    a = _vrot(np.asarray(poses, np.float64)[:, 3:7])[:, 2, :]; b = _vrot(np.asarray(gt, np.float64)[:, 3:7])[:, 2, :]
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), (a * b).sum(axis=1))
