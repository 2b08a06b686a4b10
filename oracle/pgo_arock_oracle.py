"""CPU oracle of d2pgo's ARock distributed mode (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

Restates, per agent, one pass of ARockBase::solve_arock with max_steps = 1 (d2common/src/solver/ARock.cpp:140-190) as
d2pgo_node runs it, with ARockPGO's message handling (d2pgo/src/ARockPGO.cpp:13-104):
  1. receiveAll / processPGOData: for each message (sender d, target t) in arrival order and each of its frames that the local
     problem uses: if t == self or there is no dual (d, f) yet, create it with y_l = y_r = the value, or else set y_r;
  2. scanAndCreateDualStates (:192-208): a dual (owner, f) for every frame of another agent, from x(f) (or zero);
  3. setDualStateFactors (:256-314) + the local solve: the agent's edges (and gravity priors) plus one proximal term per dual
     towards y_r, solved to convergence by pgo_lsq's sparse-direct Gauss-Newton;
  4. updateDualStates (:24-84): y_l -= eta ((y_l + y_r) / 2 - x), 4-DoF yaw normalised only outside [-pi, pi];
  5. broadcastData: one message per neighbour, target = that neighbour, the y_l of its duals.
Dual coordinates: 4-DoF [x y z yaw] (POSE_4D); 6-DoF [p ; theta], theta = Log(q_init^-1 q) (POSE_PERTURB_6D).  Proximal terms:
4-DoF ConsenusPoseFactor4D(y, rho_T, rho_theta, norm_yaw): r = diag(rho_T I3, rho_theta) [y_p - p ; N(N(y_yaw) - yaw)];
6-DoF ceres::NormalPrior(A, y), A = diag(sqrt(rho_T) I3, sqrt(rho_theta) I3): r = A ([p ; theta] - y), with the tangent
Jacobian A blockdiag(I3, J_r^-1(theta)) of the right perturbation q (x) Exp(dtheta).  arock_run is the synchronous schedule
(every agent steps, then every message goes to every other agent).  The dual table is ordered by (neighbour, frame id)."""
import numpy as np

from d2slam_b200 import synth
from oracle.pgo4d_oracle import edges_eval_4d
from oracle.pgo_gravity_oracle import priors_eval
from oracle.pgo_lsq import gauss_newton, normalize_angle
from oracle.pgo_oracle import _vqmul, _vskew, edges_eval


def theta_of(q, q_init):
    """theta = Log(q_init^-1 q), principal, and J_r^-1(theta) (the device's arock_theta, batched): q, q_init [K,4] -> [K,3], [K,3,3]."""
    q = np.asarray(q, np.float64).reshape(-1, 4); qi = np.asarray(q_init, np.float64).reshape(-1, 4)
    e = _vqmul(qi * np.array([-1.0, -1.0, -1.0, 1.0]), q)
    e = np.where(e[:, 3:4] < 0.0, -e, e)
    n = np.sqrt((e[:, :3] ** 2).sum(1))
    a = 2.0 * np.arctan2(n, e[:, 3])
    k = np.where(n > 0.0, a / np.where(n > 0.0, n, 1.0), 2.0 / e[:, 3])
    th = k[:, None] * e[:, :3]
    a2 = a * a
    with np.errstate(divide="ignore", invalid="ignore"):
        c2 = np.where(a < 1e-2, 1.0 / 12.0 + a2 / 720.0 + a2 * a2 / 30240.0, 1.0 / a2 - e[:, 3] / (2.0 * a * n))
    K = _vskew(th)
    Jinv = np.eye(3)[None] + 0.5 * K + c2[:, None, None] * np.einsum("kij,kjl->kil", K, K)
    return th, Jinv


def coords(x, q_init=None):
    """Poses in dual coordinates: [N,4] 4-DoF poses as they are; [N,7] 6-DoF poses -> [p ; theta] with q_init [N,4]."""
    x = np.asarray(x, np.float64)
    if x.shape[1] == 4:
        return x.copy()
    return np.concatenate([x[:, :3], theta_of(x[:, 3:7], q_init)[0]], axis=1)


def prox_eval(x, q_init, y, rho_T, rho_theta):
    """Proximal terms at poses x [K, 4 or 7] towards y [K, D]: r [K, D], J [K, D, D] (tangent Jacobian)."""
    x = np.asarray(x, np.float64); y = np.asarray(y, np.float64); K = len(x)
    if x.shape[1] == 4:
        r = np.empty((K, 4))
        r[:, :3] = rho_T * (y[:, :3] - x[:, :3])
        r[:, 3] = rho_theta * normalize_angle(normalize_angle(y[:, 3]) - x[:, 3])
        J = np.zeros((K, 4, 4)); J[:, [0, 1, 2], [0, 1, 2]] = -rho_T; J[:, 3, 3] = -rho_theta
        return r, J
    wT, wR = np.sqrt(rho_T), np.sqrt(rho_theta)
    th, Jinv = theta_of(x[:, 3:7], q_init)
    r = np.concatenate([wT * (x[:, :3] - y[:, :3]), wR * (th - y[:, 3:])], axis=1)
    J = np.zeros((K, 6, 6)); J[:, [0, 1, 2], [0, 1, 2]] = wT; J[:, 3:, 3:] = wR * Jinv
    return r, J


def update_duals(yl, yr, c, eta):
    """updateDualStates (ARock.cpp:50-81) in the reference's operation order; 4-DoF: yaw normalised only outside [-pi, pi]."""
    yl = np.asarray(yl, np.float64); yr = np.asarray(yr, np.float64)
    avg = (yl + yr) / 2
    out = yl - (avg - c) * eta
    if out.shape[-1] == 4:
        w = (out[..., 3] > np.pi) | (out[..., 3] < -np.pi)
        out[..., 3] = np.where(w, normalize_angle(out[..., 3]), out[..., 3])
    return out


def local_solve(x, fixed, ea, eb, rel, S, dual_pose, q_init_d, yr, rho_T, rho_theta, priors=None, iters=50, ftol=1e-15):
    """Gauss-Newton with a sparse direct solve over the edges, the gravity priors (6-DoF; priors = (idx, u_ego, S3)) and the
    proximal terms (dual k on pose dual_pose[k] towards yr[k]); to convergence.  Returns (poses, costs)."""
    x = np.asarray(x, np.float64); D = 4 if x.shape[1] == 4 else 6
    ea = np.asarray(ea); eb = np.asarray(eb); rel = np.asarray(rel, np.float64); S = np.asarray(S, np.float64).reshape(-1, D, D)
    dual_pose = np.asarray(dual_pose, int)

    def blocks(x):
        r_e, J0, J1 = (edges_eval_4d if D == 4 else edges_eval)(x, ea, eb, rel, S)
        out = [(r_e, [(ea, J0), (eb, J1)])]
        if priors is not None and len(priors[0]):
            r_g, Jg = priors_eval(x, priors[0], priors[1], priors[2])
            out.append((r_g, [(np.asarray(priors[0]), Jg)]))
        if len(dual_pose):
            r_k, J_k = prox_eval(x[dual_pose], q_init_d, yr, rho_T, rho_theta)
            out.append((r_k, [(dual_pose, J_k)]))
        return out
    return gauss_newton(x, fixed, blocks, iters, ftol)


class OracleAgent:
    """One ARock agent on the CPU.  split: pgo.arock_split output; q_init [n, 4] (6-DoF; None = the split's attitudes);
    priors: (pose index [G], u_ego [G,3], S [G,3,3]) gravity priors (6-DoF) or None."""

    def __init__(self, split, q_init=None, priors=None, rho_frame_T=0.1, rho_frame_theta=0.1, eta_k=0.9, dual_state_init_to_zero=False):
        self.split = split; self.self_id = int(split["self_id"])
        self.x = np.array(split["poses"], np.float64); self.D = 4 if self.x.shape[1] == 4 else 6
        self.ids = np.asarray(split["ids"]); self.pos = {int(i): k for k, i in enumerate(self.ids)}
        self.owner = np.asarray(split["owner"]); self.fixed = np.asarray(split["fixed"])
        self.ea = np.array([self.pos[int(i)] for i in split["id_a"]], int); self.eb = np.array([self.pos[int(i)] for i in split["id_b"]], int)
        self.qi = None if self.D == 4 else (self.x[:, 3:7] / np.linalg.norm(self.x[:, 3:7], axis=1, keepdims=True) if q_init is None else
                                             np.asarray(q_init, np.float64) / np.linalg.norm(q_init, axis=1, keepdims=True))
        self.priors = priors
        self.rho_T, self.rho_theta, self.eta, self.zero = rho_frame_T, rho_frame_theta, eta_k, bool(dual_state_init_to_zero)
        self.duals = {}            # (neighbour, frame id) -> [y_l, y_r]
        self.inbox = []
        self.in_problem = np.zeros(len(self.ids), bool); self.in_problem[self.ea] = True; self.in_problem[self.eb] = True
        if priors is not None:
            self.in_problem[np.asarray(priors[0], int)] = True
        self.last_costs = None
        self.replay = None         # an iterator of local solutions (poses [n, 4 or 7]) in place of the local solve, or None

    def receive(self, msg):
        self.inbox.append(msg)

    def _process(self):
        for sender, target, frames, vals in self.inbox:
            for f, v in zip(frames, np.asarray(vals, np.float64).reshape(len(frames), -1)):
                i = self.pos.get(int(f))
                if i is None or not self.in_problem[i]:
                    continue
                key = (int(sender), int(f))
                if target == self.self_id or key not in self.duals:
                    if key not in self.duals:
                        self.duals[key] = [v.copy(), v.copy()]
                    else:
                        self.duals[key][1] = v.copy()
        self.inbox = []

    def _scan(self):
        c = coords(self.x, self.qi)
        for i, f in enumerate(self.ids):
            o = int(self.owner[i])
            if not self.in_problem[i] or o == self.self_id or (o, int(f)) in self.duals:
                continue
            v = np.zeros(self.D) if self.zero else c[i].copy()
            self.duals[(o, int(f))] = [v.copy(), v.copy()]

    def table(self):
        """keys in table order, pose index per dual, y_l [K, D], y_r [K, D]"""
        keys = sorted(self.duals)
        idx = np.array([self.pos[f] for _, f in keys], int)
        yl = np.array([self.duals[k][0] for k in keys]).reshape(-1, self.D); yr = np.array([self.duals[k][1] for k in keys]).reshape(-1, self.D)
        return keys, idx, yl, yr

    def terms(self):
        """r | J of every dual's proximal term at the current poses, [K, D + D^2] (d2pgo_debug_arock_terms' layout)."""
        keys, idx, yl, yr = self.table()
        r, J = prox_eval(self.x[idx], None if self.qi is None else self.qi[idx], yr, self.rho_T, self.rho_theta)
        return np.concatenate([r, J.reshape(len(keys), -1)], axis=1)

    def step(self):
        self._process()
        self._scan()
        keys, idx, yl, yr = self.table()
        if self.replay is not None:
            self.x = np.array(next(self.replay), np.float64)
        else:
            self.x, self.last_costs = local_solve(self.x, self.fixed, self.ea, self.eb, self.split["rel"], self.split["sqrt_info"], idx,
                                                  None if self.qi is None else self.qi[idx], yr, self.rho_T, self.rho_theta, self.priors)
        if keys:
            yl = update_duals(yl, yr, coords(self.x[idx], None if self.qi is None else self.qi[idx]), self.eta)
            for k, key in enumerate(keys):
                self.duals[key][0] = yl[k]

    def messages(self):
        keys = sorted(self.duals)
        out = []
        for n in sorted({k[0] for k in keys}):
            fs = [f for m, f in keys if m == n]
            out.append((self.self_id, n, np.array(fs, np.int64), np.array([self.duals[(n, f)][0] for f in fs])))
        return out


def arock_run(agents, rounds, after_round=None):
    """pgo.arock_run's synchronous schedule for OracleAgent lists."""
    for r in range(rounds):
        for a in agents:
            a.step()
        msgs = [m for a in agents for m in a.messages()]
        for a in agents:
            for m in msgs:
                if m[0] != a.self_id:
                    a.receive(m)
        if after_round is not None:
            after_round(r, agents)


def copy_disagreement(agents):
    """Largest difference between two agents' copies of one frame: (position [m], rotation / yaw [rad])."""
    seen = {}
    for a in agents:
        for i, f in enumerate(a.ids):
            seen.setdefault(int(f), []).append(a.x[i])
    dp = dr = 0.0
    for xs in seen.values():
        for u in xs[1:]:
            v = xs[0]
            dp = max(dp, float(np.linalg.norm(u[:3] - v[:3])))
            if len(u) == 4:
                dr = max(dr, float(abs(normalize_angle(u[3] - v[3]))))
            else:
                dr = max(dr, float(synth.pose_errors(u[None], v[None])[1]))
    return dp, dr
