"""CPU oracle of the pose graph's LM loop with exact steps (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

Restates pgo_solve of d2slam_b200/csrc/d2pgo.cu with the linear solve replaced by scipy's sparse direct solver, which is what
the sparse-Cholesky path (d2pgo_set_linear_solver(h, D2PGO_LINEAR_SPARSE_CHOLESKY)) computes on the device:
  step      (J^T J + diag(lambda d + 1e-12)) dx = -J^T r over the free poses, d = the diagonal of the block diagonal the device
            forms per pose (sum over the pose's edge sides J_side^T J_side, plus its gravity prior): a self loop's cross terms
            are in J^T J but not in d
  accept    cand < cost (and finite): lambda = max(lambda / 3, 1e-12) (0 stays 0), stop when the relative decrease is below
            function_tolerance
  reject    lambda = 4 lambda (1e-4 from 0), stop above 1e8
Factors: RelPoseFactorAD (pgo_oracle.edges_eval), RelPoseFactor4D (pgo4d_oracle.edges_eval_4d) and the gravity prior
(pgo_gravity_oracle.priors_eval), each pinned to the reference elsewhere."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import pgo4d_oracle as p4
from oracle import pgo_gravity_oracle as pg
from oracle import pgo_lsq
from oracle import pgo_oracle as po


class Problem:
    """One pose graph: poses [N, 7] (6-DoF) or [N, 4] (4-DoF), fixed flags, edges, optional 6-DoF gravity priors
    (idx [G] pose indices, u_ego [G, 3], S [G, 3, 3])."""

    def __init__(self, poses, fixed, ea, eb, rel, sqrt_info, prior_idx=None, prior_u=None, prior_S=None):
        self.x0 = np.array(poses, np.float64)
        self.D = 4 if self.x0.shape[1] == 4 else 6
        self.fixed = np.asarray(fixed) != 0
        self.ea = np.asarray(ea); self.eb = np.asarray(eb); self.rel = np.asarray(rel, np.float64)
        self.S = np.asarray(sqrt_info, np.float64).reshape(-1, self.D, self.D)
        self.pidx = np.zeros(0, int) if prior_idx is None else np.asarray(prior_idx, int)
        self.pu = None if prior_u is None else np.asarray(prior_u, np.float64).reshape(-1, 3)
        self.pS = None if prior_S is None else np.asarray(prior_S, np.float64).reshape(-1, 3, 3)
        self.free, self.col = pgo_lsq.free_columns(self.fixed, self.D)

    def system(self, x):
        """residual r, sparse J over the free tangents, and d (the diagonal the damping scales)."""
        r_e, J0, J1 = (p4.edges_eval_4d if self.D == 4 else po.edges_eval)(x, self.ea, self.eb, self.rel, self.S)
        blocks = [(r_e, [(self.ea, J0), (self.eb, J1)])]
        if len(self.pidx):
            r_g, Jg = pg.priors_eval(x, self.pidx, self.pu, self.pS)
            blocks.append((r_g, [(self.pidx, Jg)]))
        return pgo_lsq.assemble(blocks, self.col, len(self.free), self.D, diag=True)

    def cost(self, x):
        r = self.system(x)[0]
        return 0.5 * float(r @ r)

    def retract(self, x, dx):
        return pgo_lsq.retract(x, self.free, dx)

    def step(self, x, lam):
        """The exact step dx [N, D] (0 on fixed poses)."""
        r, J, d = self.system(x)
        H = (J.T @ J).tocsc() + sp.diags(lam * d + 1e-12, format="csc")
        dx = spla.spsolve(H, -(J.T @ r)) if H.shape[0] else np.zeros(0)
        out = np.zeros((len(x), self.D)); out[self.free] = dx.reshape(-1, self.D)
        return out


def lm_solve(prob, max_iterations=20, lambda0=1e-6, function_tolerance=1e-9):
    """The device's LM loop with exact steps.  Returns (x, history, report) with history = [(candidate cost, accepted)] per
    iteration and report = dict(iterations, accepted, converged, initial_cost, final_cost)."""
    x = prob.x0.copy()
    cost = prob.cost(x); lam = lambda0
    hist = []; rep = dict(iterations=0, accepted=0, converged=0, initial_cost=cost)
    for _ in range(max_iterations):
        cand_x = prob.retract(x, prob.step(x, lam)[prob.free])
        cand = prob.cost(cand_x)
        rep["iterations"] += 1
        ok = cand < cost and np.isfinite(cand)
        hist.append((cand, bool(ok)))
        if ok:
            rel_dec = (cost - cand) / (cost if cost > 0 else 1.0)
            x = cand_x; cost = cand; rep["accepted"] += 1
            lam = max(lam / 3.0, 1e-12) if lam > 0 else 0.0
            if rel_dec < function_tolerance:
                rep["converged"] = 1
                break
        else:
            lam = lam * 4.0 if lam > 0 else 1e-4
            if lam > 1e8:
                break
    rep["final_cost"] = cost
    return x, hist, rep
