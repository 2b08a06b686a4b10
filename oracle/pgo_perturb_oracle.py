"""CPU oracle of the pose graph's perturbation chart (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

d2pgo's 6-DoF node runs in perturb_mode (d2pgo/src/d2pgo_node.cpp:216; include/d2pgo.h d2pgo_set_chart): the parameter block of
frame f is the Euclidean 6-vector x_f = [p_f, theta_f] (POSE_PERTURB_6D, no manifold) and its attitude is

    q_f = q_init,f (x) quatfromRotationVector(theta_f)       (utils.hpp:39-55: [theta / 2, 1] unnormalised if |theta| < 1e-2,
                                                              else the exact exponential; quaternions [x y z w] here)

The factors, as the reference writes them (RelPoseFactorPerturbAD, RelPoseFactor.hpp:138-195; GravityPriorPerturbAD,
GravityPrior.hpp:8-46):

    relative pose   q_c = q_a.conjugate() = (v, w), t = p_b - p_a, uv = 2 v x t,
                    p_ab = t + w uv + v x uv                    (Eigen's _transformVector: not a rotation for a non-unit q_a)
                    dq = q_meas (x) (q_c (x) q_b).conjugate(),  r = S [p_ab - p_meas ; 2 vec(dq)]
    gravity prior   u = row 2 of q_a.toRotationMatrix() = [2 (xz - yw), 2 (yz + xw), 1 - 2 (x^2 + y^2)],  r = S^T (u - u_ego)

with analytic Jacobians in [p, theta] (what ceres' dual numbers give: inside the ball d dq / d theta = [I / 2 ; 0]).  Factor
level PINNED: relpose_eval / gravity_eval against the reference's own functors compiled into oracle/_ref/libd2ref_gravity.so
(tests/test_pgo_perturb_oracle.py, tests/golden/ref_perturb.npz).  ChartProblem restates a chart problem in the interface of
pgo_ceres_lm_oracle.ceres_lm_solve (x + dx retraction, 6-vector norms); solve_chart is a Gauss-Newton to convergence on it.
NodeState restates the node's persistent state across solves (PGOState::addFrame, postPerturbSolve, recoverRotationLLT);
arock_agent is the chart form of pgo_ceres_lm_oracle.arock_agent (ARockPGO in perturb mode, ARockPGO.cpp:21-23)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import pgo_lsq
from oracle.pgo_ceres_lm_oracle import BlocksProblem
from oracle.pgo_gravity_oracle import ego_gravity

EPS = 1e-2   # quatfromRotationVector's ball


def _skew(v):
    v = np.asarray(v, np.float64)
    K = np.zeros(v.shape[:-1] + (3, 3))
    K[..., 0, 1] = -v[..., 2]; K[..., 0, 2] = v[..., 1]; K[..., 1, 0] = v[..., 2]
    K[..., 1, 2] = -v[..., 0]; K[..., 2, 0] = -v[..., 1]; K[..., 2, 1] = v[..., 0]
    return K


def qmul(a, b):
    """Hamilton product a (x) b of [..., 4] quaternions [x y z w], Eigen's formulas."""
    ax, ay, az, aw = np.moveaxis(np.asarray(a, np.float64), -1, 0)
    bx, by, bz, bw = np.moveaxis(np.asarray(b, np.float64), -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def qconj(q):
    q = np.array(q, np.float64)
    q[..., :3] *= -1.0
    return q


def qL(q):
    """L(q) [..., 4, 4]: q (x) p = L(q) p"""
    x, y, z, w = np.moveaxis(np.asarray(q, np.float64), -1, 0)
    return np.stack([np.stack([w, -z, y, x], -1), np.stack([z, w, -x, y], -1), np.stack([-y, x, w, z], -1),
                     np.stack([-x, -y, -z, w], -1)], -2)


def qR(q):
    """R(q) [..., 4, 4]: p (x) q = R(q) p"""
    x, y, z, w = np.moveaxis(np.asarray(q, np.float64), -1, 0)
    return np.stack([np.stack([w, z, -y, x], -1), np.stack([-z, w, x, y], -1), np.stack([y, -x, w, z], -1),
                     np.stack([-x, -y, -z, w], -1)], -2)


def quat_from_rotation_vector(theta):
    """quatfromRotationVector [..., 3] -> (dq [..., 4], d dq / d theta [..., 4, 3]); the branch on sqrt(theta . theta)."""
    th = np.asarray(theta, np.float64)
    n = np.sqrt(th[..., 0] * th[..., 0] + th[..., 1] * th[..., 1] + th[..., 2] * th[..., 2])
    ball = n < EPS
    ns = np.where(ball, 1.0, n)
    h = ns / 2.0; s = np.sin(h); c = np.cos(h)
    u = th / ns[..., None]
    q = np.concatenate([u * s[..., None], c[..., None]], axis=-1)
    J = np.zeros(th.shape[:-1] + (4, 3))
    J[..., :3, :] = (s / ns)[..., None, None] * (np.eye(3) - u[..., :, None] * u[..., None, :]) + (0.5 * c)[..., None, None] * u[..., :, None] * u[..., None, :]
    J[..., 3, :] = -0.5 * s[..., None] * u
    qb = np.concatenate([th / 2.0, np.ones(th.shape[:-1] + (1,))], axis=-1)
    Jb = np.zeros_like(J); Jb[..., 0, 0] = Jb[..., 1, 1] = Jb[..., 2, 2] = 0.5
    return np.where(ball[..., None], qb, q), np.where(ball[..., None, None], Jb, J)


def attitude(x6, qi):
    """q = q_init (x) dq(theta) (not normalised) and d q / d theta [..., 4, 3]."""
    x6 = np.asarray(x6, np.float64); qi = np.asarray(qi, np.float64)
    dq, Jd = quat_from_rotation_vector(x6[..., 3:6])
    return qmul(qi, dq), qL(qi) @ Jd


def relpose_eval(xa, xb, qia, qib, rel7, S):
    """RelPoseFactorPerturbAD for E edges: xa, xb [E, 6], qia, qib [E, 4], rel7 [E, 7], S [E, 6, 6] -> r [E, 6], Ja, Jb [E, 6, 6]."""
    xa = np.atleast_2d(np.asarray(xa, np.float64)); xb = np.atleast_2d(np.asarray(xb, np.float64))
    rel = np.atleast_2d(np.asarray(rel7, np.float64)); S = np.asarray(S, np.float64).reshape(-1, 6, 6)
    qa, Jqa = attitude(xa, np.atleast_2d(qia)); qb, Jqb = attitude(xb, np.atleast_2d(qib))
    qc = qconj(qa); qm = rel[:, 3:7]
    t = xb[:, :3] - xa[:, :3]; v = qc[:, :3]; w = qc[:, 3]
    uv = 2.0 * np.cross(v, t)
    pab = t + w[:, None] * uv + np.cross(v, uv)
    dq = qmul(qm, qconj(qmul(qc, qb)))
    raw = np.concatenate([pab - rel[:, :3], 2.0 * dq[:, :3]], axis=1)
    r = np.einsum("eij,ej->ei", S, raw)
    Vx, Tx = _skew(v), _skew(t)
    M = np.eye(3) + 2.0 * w[:, None, None] * Vx + 2.0 * Vx @ Vx
    Pq = np.zeros((len(xa), 3, 4))
    Pq[:, :, :3] = -(-2.0 * w[:, None, None] * Tx - _skew(uv) - 2.0 * Vx @ Tx)
    Pq[:, :, 3] = uv
    C = np.diag([-1.0, -1.0, -1.0, 1.0])
    Da = (qL(qm) @ C @ qR(qb) @ C)[:, :3, :]
    Db = (qL(qm) @ C @ qL(qc))[:, :3, :]
    A0 = np.zeros((len(xa), 6, 6)); A1 = np.zeros((len(xa), 6, 6))
    A0[:, :3, :3] = -M; A1[:, :3, :3] = M
    A0[:, :3, 3:] = Pq @ Jqa; A0[:, 3:, 3:] = 2.0 * Da @ Jqa; A1[:, 3:, 3:] = 2.0 * Db @ Jqb
    return r, S @ A0, S @ A1


def gravity_eval(x6, qi, u_ego, S):
    """GravityPriorPerturbAD for G priors: x6 [G, 6], qi [G, 4], u_ego [G, 3] (ego_gravity), S [G, 3, 3] -> r [G, 3], J [G, 3, 6]."""
    x6 = np.atleast_2d(np.asarray(x6, np.float64)); S = np.asarray(S, np.float64).reshape(-1, 3, 3)
    q, Jq = attitude(x6, np.atleast_2d(qi))
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    u = np.stack([tz * x - ty * w, tz * y + tx * w, 1 - (tx * x + ty * y)], axis=1)   # Eigen's toRotationMatrix, row 2
    St = np.transpose(S, (0, 2, 1))
    r = np.einsum("gij,gj->gi", St, u - np.asarray(u_ego, np.float64).reshape(-1, 3))
    U = np.stack([np.stack([2 * z, -2 * w, 2 * x, -2 * y], -1), np.stack([2 * w, 2 * z, 2 * y, 2 * x], -1),
                  np.stack([-4 * x, -4 * y, 0 * x, 0 * x], -1)], -2)
    J = np.zeros((len(x6), 3, 6))
    J[:, :, 3:] = St @ U @ Jq
    return r, J


def poses_of(x, qinit):
    """[p, normalise(q_init (x) dq(theta))] of chart states x [N, 6] (d2pgo_get_poses on a chart handle)."""
    q = attitude(x, qinit)[0]
    return np.concatenate([np.asarray(x, np.float64)[:, :3], q / np.linalg.norm(q, axis=1, keepdims=True)], axis=1)


def enter(poses7):
    """PGOState::addFrame in the chart: x = [p, 0], q_init = the normalised attitude."""
    p = np.asarray(poses7, np.float64)
    x = np.zeros((len(p), 6)); x[:, :3] = p[:, :3]
    return x, p[:, 3:7] / np.linalg.norm(p[:, 3:7], axis=1, keepdims=True)


def prox_eval(x6, yr, rho_T, rho_theta):
    """ARock's proximal NormalPrior in the chart (ARock.cpp:284-291): the dual coordinates are the state, so
    r = diag(sqrt(rho_T) I3, sqrt(rho_theta) I3) (x - y_r) with that constant diagonal as J; x6, yr [K, 6] -> r [K, 6], J [K, 6, 6]"""
    x6 = np.asarray(x6, np.float64); yr = np.asarray(yr, np.float64).reshape(-1, 6)
    w = np.r_[np.full(3, np.sqrt(rho_T)), np.full(3, np.sqrt(rho_theta))]
    return w * (x6 - yr), np.tile(np.diag(w), (len(x6), 1, 1))


class ChartProblem(BlocksProblem):
    """A chart problem for pgo_ceres_lm_oracle.ceres_lm_solve: states x0 [N, 6], q_init [N, 4], fixed flags, edges (pose indices
    ea, eb, rel7 [E, 7], S [E, 6, 6]), gravity priors (pose index idx [G], ego poses [G, 7] or u_ego [G, 3], S [G, 3, 3]) and ARock proximal
    terms (prox = (pose index [K], y_r [K, 6], rho_T, rho_theta): prox_eval); x + dx retraction."""

    def __init__(self, x0, qinit, fixed, ea, eb, rel, S, prior_idx=(), ego7=None, prior_S=None, prox=None, u_ego=None):
        self.qinit = np.asarray(qinit, np.float64)
        ea = np.asarray(ea, int); eb = np.asarray(eb, int); rel = np.asarray(rel, np.float64); S = np.asarray(S, np.float64).reshape(-1, 6, 6)
        gi = np.asarray(prior_idx, int)
        ue = (ego_gravity(ego7) if ego7 is not None else np.asarray(u_ego, np.float64)) if len(gi) else None
        gS = None if not len(gi) else np.asarray(prior_S, np.float64).reshape(-1, 3, 3)
        qi = self.qinit

        def blocks(x):
            r, Ja, Jb = relpose_eval(x[ea], x[eb], qi[ea], qi[eb], rel, S)
            out = [(r, [(ea, Ja), (eb, Jb)])]
            if len(gi):
                rg, Jg = gravity_eval(x[gi], qi[gi], ue, gS)
                out.append((rg, [(gi, Jg)]))
            if prox is not None and len(prox[0]):
                rk, Jk = prox_eval(x[prox[0]], prox[1], prox[2], prox[3])
                out.append((rk, [(np.asarray(prox[0], int), Jk)]))
            return out
        super().__init__(np.asarray(x0, np.float64), fixed, blocks)

    def retract(self, x, dx):
        y = x.copy()
        y[self.free] += np.asarray(dx).reshape(-1, 6)
        return y

    def gradient(self, x):
        r, J = pgo_lsq.assemble(self.blocks_at(x), self.col, len(self.free), 6)
        return J.T @ r


def solve_chart(prob, iters=60, ftol=1e-15):
    """Gauss-Newton with a sparse direct solve in the chart to convergence; returns (x, costs)."""
    x = prob.x0.copy()
    costs = []
    for it in range(iters):
        r, J = pgo_lsq.assemble(prob.blocks_at(x), prob.col, len(prob.free), 6)
        c = 0.5 * float(r @ r); costs.append(c)
        if it and abs(costs[-2] - c) <= ftol * max(c, 1e-300):
            break
        H = (J.T @ J).tocsc(); g = J.T @ r
        x = prob.retract(x, spla.spsolve(H + 1e-12 * sp.identity(H.shape[0], format="csc"), -g))
    return x, costs


class NodeState:
    """The node's chart state across solves, keyed by frame id: x [p, theta] and q_init per frame (d2pgo_set_chart /
    d2pgo_set_poses / d2pgo_rot_init on a chart handle)."""

    def __init__(self, ids, poses7):
        x, q = enter(poses7)
        self.x = {int(i): x[k] for k, i in enumerate(ids)}
        self.q = {int(i): q[k] for k, i in enumerate(ids)}

    def set_poses(self, ids, poses7):
        """present ids keep x and q_init, new ones start at [p, 0] with their attitude; ids not listed are dropped"""
        x, q = enter(poses7)
        self.x = {int(i): self.x.get(int(i), x[k]) for k, i in enumerate(ids)}
        self.q = {int(i): self.q.get(int(i), q[k]) for k, i in enumerate(ids)}

    def arrays(self, ids):
        return np.array([self.x[int(i)] for i in ids]), np.array([self.q[int(i)] for i in ids])

    def poses(self, ids):
        return poses_of(*self.arrays(ids))

    def rot_init(self, ids, poses7_after):
        """q_init = the attitude after rotation initialisation run on poses(ids) (initialised or current); x untouched"""
        q = np.asarray(poses7_after, np.float64)[:, 3:7]
        for k, i in enumerate(ids):
            self.q[int(i)] = q[k] / np.linalg.norm(q[k])

    def solve(self, ids, fixed, ea, eb, rel, S, solver, **kw):
        """one solve from the kept state; solver(prob, **kw) -> (x, ...); the state keeps the result"""
        x, q = self.arrays(ids)
        out = solver(ChartProblem(x, q, fixed, ea, eb, rel, S), **kw)
        for k, i in enumerate(ids):
            self.x[int(i)] = out[0][k]
        return out


def arock_agent(split, lm_cfg=None, q_init=None, **kw):
    """pgo_ceres_lm_oracle.arock_agent in the chart: a pgo_arock_oracle.OracleAgent whose state is [p, theta] per frame (entered
    from the split's poses, q_init [n, 4] or their attitudes), whose duals are that state (no log map), whose proximal terms are
    prox_eval and whose local solves run ceres_lm_solve(**lm_cfg) on a ChartProblem.  .x is the state [n, 6], .qc its q_init,
    .poses() the poses [n, 7] (d2pgo_get_poses).  kw: OracleAgent's arguments."""
    from oracle import pgo_arock_oracle as pa
    from oracle.pgo_ceres_lm_oracle import ceres_lm_solve

    class ChartAgent(pa.OracleAgent):
        def __init__(self):
            super().__init__(split, **kw)
            self.x, self.qc = enter(split["poses"])
            if q_init is not None:
                self.qc = np.asarray(q_init, np.float64) / np.linalg.norm(q_init, axis=1, keepdims=True)

        def _scan(self):   # OracleAgent._scan with the state as the dual coordinates
            for i, f in enumerate(self.ids):
                o = int(self.owner[i])
                if not self.in_problem[i] or o == self.self_id or (o, int(f)) in self.duals:
                    continue
                v = np.zeros(6) if self.zero else self.x[i].copy()
                self.duals[(o, int(f))] = [v.copy(), v.copy()]

        def terms(self):
            keys, idx, yl, yr = self.table()
            r, J = prox_eval(self.x[idx], yr, self.rho_T, self.rho_theta)
            return np.concatenate([r, J.reshape(len(keys), -1)], axis=1)

        def poses(self):
            return poses_of(self.x, self.qc)

        def step(self):   # process, scan, the ceres solve in the chart, updateDualStates on the state
            self._process()
            self._scan()
            keys, idx, yl, yr = self.table()
            pri = {} if self.priors is None else dict(prior_idx=self.priors[0], u_ego=self.priors[1], prior_S=self.priors[2])
            prob = ChartProblem(self.x, self.qc, self.fixed, self.ea, self.eb, self.split["rel"], self.split["sqrt_info"], **pri,
                                prox=(idx, yr, self.rho_T, self.rho_theta))
            self.x, _, rep = ceres_lm_solve(prob, **(lm_cfg or {}))
            self.last_costs = [rep["initial_cost"], rep["final_cost"]]
            if keys:
                yl = pa.update_duals(yl, yr, self.x[idx], self.eta)
                for k, key in enumerate(keys):
                    self.duals[key][0] = yl[k]
    return ChartAgent()
