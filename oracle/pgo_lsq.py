"""Sparse least squares shared by the pose-graph CPU oracles (TEST INFRASTRUCTURE: imported by those oracles only).

A problem is a list of residual blocks (r [M, D'], [(pose index [M], J [M, D', D]), ...]): M residuals of D' rows each, and per
part the Jacobian of every residual with respect to the D-dimensional tangent of one pose.  The blocks stack in list order into
one residual vector; the Jacobian's columns are the tangents of the free poses, in pose order.  The factors live in the oracle
modules, which import this one; it imports none of them."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from d2slam_b200 import synth


def normalize_angle(a):
    """Utility::NormalizeAngle (utils.hpp:251-257)"""
    return a - 2.0 * np.pi * np.floor((a + np.pi) / (2.0 * np.pi))


def free_columns(fixed, D):
    """The free poses' indices and col [N]: each free pose's first tangent column (0, D, 2D, ... in pose order), -1 if fixed."""
    fixed = np.asarray(fixed)
    free = np.nonzero(fixed == 0)[0]; col = -np.ones(len(fixed), int); col[free] = np.arange(len(free)) * D
    return free, col


def assemble(blocks, col, n_free, D, diag=False):
    """The stacked residual r and the CSR Jacobian J [len(r), D n_free] of the blocks (fixed poses' parts dropped).  With diag,
    also d [D n_free], the diagonal of sum over parts of J_part^T J_part, so a self loop's cross terms are in J^T J but not in d."""
    rows, cols, vals, res = [], [], [], []
    d = np.zeros(D * n_free) if diag else None
    off = 0
    for r_b, parts in blocks:
        m, dr = r_b.shape
        rb, cb = np.meshgrid(np.arange(dr), np.arange(D), indexing="ij")
        for idx, J in parts:
            keep = col[idx] >= 0
            e_idx = np.nonzero(keep)[0]; c = col[idx[keep]]; Jk = J[keep]
            rows.append((off + dr * e_idx[:, None, None] + rb[None]).ravel()); cols.append((c[:, None, None] + cb[None]).ravel()); vals.append(Jk.ravel())
            if diag:
                np.add.at(d, (c[:, None] + np.arange(D)[None]).ravel(), (Jk ** 2).sum(axis=1).ravel())
        res.append(r_b.ravel()); off += m * dr
    J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(off, D * n_free))
    return (np.concatenate(res), J, d) if diag else (np.concatenate(res), J)


def retract(x, free, dx):
    """A copy of the poses x [N, 4 or 7] with the free ones moved by dx (n_free tangents of D): 4-DoF PosAngleManifold::Plus
    (angle_manifold.h:39-68: x + dx, yaw normalised to [-pi, pi)), 6-DoF synth.pose_plus one pose at a time."""
    y = x.copy()
    if x.shape[1] == 4:
        dx = dx.reshape(-1, 4)
        y[free, :3] += dx[:, :3]
        y[free, 3] = normalize_angle(y[free, 3] + dx[:, 3])
    else:
        dx = dx.reshape(-1, 6)
        for k, i in enumerate(free):
            y[i] = synth.pose_plus(x[i], dx[k])
    return y


def gauss_newton(x0, fixed, blocks_at, iters, ftol):
    """Gauss-Newton with a sparse direct solve over the free poses of x0 [N, 4 or 7]; blocks_at(x) gives the residual blocks at
    poses x.  Each of at most iters iterations evaluates the cost, then steps; it stops before the step when the cost changed by at
    most ftol relative to the previous one.  Returns (poses, costs)."""
    x = np.array(x0, np.float64); D = 4 if x.shape[1] == 4 else 6
    free, col = free_columns(fixed, D)
    costs = []
    for it in range(iters):
        r, J = assemble(blocks_at(x), col, len(free), D)
        c = 0.5 * float(r @ r); costs.append(c)
        if it and abs(costs[-2] - c) <= ftol * max(c, 1e-300):
            break
        H = (J.T @ J).tocsc(); g = J.T @ r
        x = retract(x, free, spla.spsolve(H + 1e-12 * sp.identity(H.shape[0], format="csc"), -g))
    return x, costs
