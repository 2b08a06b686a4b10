"""CPU oracle of the 4-DoF pose-graph path (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

The batched linearisation and the scipy sparse-direct Gauss-Newton of pgo_oracle.py for d2pgo's default configuration,
RelPoseFactor4D on [x y z yaw] poses (pgo_pose_dof = PGO_POSE_4D).  Factor level pinned: edges_eval_4d is the per-edge
pgo_oracle.edge_eval_4d batched (tests/test_pgo_4dof.py), and edge_eval_4d is pinned to the reference functor
(tests/test_ref_pin.py, tests/golden/ref_factors.npz); the minimiser is a restatement (same optimum, not ceres' iterates)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle.pgo_oracle import normalize_angle
def edges_eval_4d(poses, ea, eb, rel, S):
    """edge_eval_4d for all edges at once (same formulas, numpy-batched): poses [N,4], rel [E,4] = [p_meas, yaw_meas], S [E,4,4]
    -> r [E,4], J0 [E,4,4], J1 [E,4,4]."""
    pa, pb = poses[ea], poses[eb]
    c, s_ = np.cos(-pa[:, 3]), np.sin(-pa[:, 3])
    v = pb[:, :3] - pa[:, :3]
    E = len(ea)
    Rz = np.zeros((E, 3, 3)); Rz[:, 0, 0] = c; Rz[:, 0, 1] = -s_; Rz[:, 1, 0] = s_; Rz[:, 1, 1] = c; Rz[:, 2, 2] = 1.0
    dRz = np.zeros((E, 3, 3)); dRz[:, 0, 0] = -s_; dRz[:, 0, 1] = -c; dRz[:, 1, 0] = c; dRz[:, 1, 1] = -s_
    raw = np.concatenate([rel[:, :3] - np.einsum("eij,ej->ei", Rz, v), normalize_angle(rel[:, 3] - normalize_angle(pb[:, 3] - pa[:, 3]))[:, None]], axis=1)
    A0 = np.zeros((E, 4, 4)); A1 = np.zeros((E, 4, 4))
    A0[:, :3, :3] = Rz; A0[:, :3, 3] = np.einsum("eij,ej->ei", dRz, v); A0[:, 3, 3] = 1.0
    A1[:, :3, :3] = -Rz; A1[:, 3, 3] = -1.0
    return np.einsum("eij,ej->ei", S, raw), np.einsum("eij,ejk->eik", S, A0), np.einsum("eij,ejk->eik", S, A1)


def cost_4d(poses, ea, eb, rel, S):
    r = edges_eval_4d(np.asarray(poses, float), np.asarray(ea), np.asarray(eb), np.asarray(rel, float), np.asarray(S).reshape(-1, 4, 4))[0]
    return 0.5 * float(np.sum(r * r))


def solve_4d(poses, fixed, ea, eb, rel, sqrt_info, iters=30, ftol=1e-12):
    """solve() for the 4-DoF problem: Gauss-Newton with a sparse direct solve, retraction of PosAngleManifold::Plus
    (angle_manifold.h:39-68: x + dx, yaw normalised to [-pi, pi)); returns (poses, costs)."""
    x = np.array(poses, float); N = len(x); S = np.asarray(sqrt_info).reshape(-1, 4, 4)
    free = np.nonzero(np.asarray(fixed) == 0)[0]; col = -np.ones(N, int); col[free] = np.arange(len(free)) * 4
    costs = []
    ea = np.asarray(ea); eb = np.asarray(eb); rel = np.asarray(rel, float)
    E = len(ea); rr, cc = np.meshgrid(np.arange(4), np.arange(4), indexing="ij")
    for it in range(iters):
        r_e, J0, J1 = edges_eval_4d(x, ea, eb, rel, S)                   # == edge_eval_4d per edge (tests/test_pgo_4dof.py)
        r_all = r_e.ravel()
        rows, cols, vals = [], [], []
        for blk, J in ((ea, J0), (eb, J1)):
            keep = col[blk] >= 0
            e_idx = np.nonzero(keep)[0]
            rows.append((4 * e_idx[:, None, None] + rr[None]).ravel()); cols.append((col[blk[keep]][:, None, None] + cc[None]).ravel()); vals.append(J[keep].ravel())
        J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(4 * E, 4 * len(free)))
        c = 0.5 * float(r_all @ r_all); costs.append(c)
        if it and abs(costs[-2] - c) <= ftol * max(c, 1e-300):
            break
        H = (J.T @ J).tocsc(); g = J.T @ r_all
        dx = spla.spsolve(H + 1e-12 * sp.identity(H.shape[0], format="csc"), -g).reshape(-1, 4)
        x[free, :3] += dx[:, :3]
        x[free, 3] = normalize_angle(x[free, 3] + dx[:, 3])
    return x, costs
