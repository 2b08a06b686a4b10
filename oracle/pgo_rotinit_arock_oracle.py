"""numpy / scipy restatement of d2pgo's distributed rotation initialisation (RotationInitARock<double>,
d2pgo/src/rot_init/rotation_initialization_arock.hpp, on ARockBase::solve_arock, d2common/src/solver/ARock.cpp:140-190), the
row systems solved sparse-direct.  Checks include/d2pgo.h d2pgo_arock_rot_*.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_rotinit_arock.py and tools/pgo_rotinit_arock_bench.py.  Nothing under
d2slam_b200/ imports it.  Line numbers are those of rotation_initialization_arock.hpp unless stated; "base" is
rotation_initialization_base.hpp.

One step of an agent (RotationInitARock::solve with max_steps = 1):
  1. receiveAll / processPGOData (:104-111, :142-182): messages in arrival order; for a frame an edge names, if target == self
     or there is no dual (sender, f): the dual is created with zeros if missing, y_r = the value, y_l = the value if created;
  2. prepareSolverInIter (:74-77): the fixed-frame edge rows (base :72-87, pgo_rotinit_oracle.build_system);
  3. scanAndCreateDualStates (:79-102): every edge end another agent owns gets the dual (owner, f) = 0 if it has none;
  4. setDualStateFactors (:32-61): per dual on a free frame, w (r_f^k - (row k of Y_r)^T) = 0 with w = dual_weight(rho);
  5. solveLinearRot (base :178-213): x = (A^T A)^-1 A^T b, gravity rows for every free frame (owned or remote);
  6. recoverRotationLLT (base :360-389): state_changes = mean |R_state - M_f|_F / |R_state|_F, R_state = M_f, and only owned
     frames take the attitude of project(M_f) (the zero matrix projects to I: Eigen's JacobiSVD gives U = V = I there);
  7. updateDualStates, vector branch (ARock.cpp:63-81): y_l -= eta ((y_l + y_r) / 2 - R_state), every dual;
  8. broadcastData (:113-140): per neighbour of the table, the y_l and this agent's pose of each frame.
At receipt (inputDPGOData :216-235) the frames the sender owns take the sender's pose at once.  R_state starts as
R(attitude) when a frame first enters a step (PGOState::addFrame, pgostate.hpp:36-39).

ASSUMED (swarm_msgs is not in the reference tree): Swarm::PosePrior(id, Matrix3d M, Matrix3d info) keeps M unprojected for
getRotMat(), and info = rho I3 is information whose Cholesky factor is the square root, so w = |sqrt(rho) I3|_F = sqrt(3 rho).
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.sparse.csgraph import connected_components

from oracle.pgo_arock_oracle import update_duals
from oracle.pgo_rotinit_oracle import R_quat, build_system, project_so3, quat_R


def dual_weight(rho_rot_mat):
    """w of a dual prior PosePrior(f, Y_r, rho I3): |getSqrtInfoMatRot()|_F under the ASSUMED convention above."""
    return float(np.sqrt(3.0 * rho_rot_mat))


def project(M):
    """recoverRotationSVD of one 3x3 M, with JacobiSVD's U = V = I on the zero matrix."""
    M = np.asarray(M, np.float64)
    return np.eye(3) if not M.any() else project_so3(M)


class RotAgent:
    """One agent of the distributed rotation initialisation.  split: pgo.arock_split output (6-DoF); ego_poses [n, 7] of the
    split's frames (gravity rows only).  Exposes the ArockAgent method names rot_init_step / rot_messages / rot_receive, so that
    pgo.arock_rot_init_run drives it too."""

    def __init__(self, split, eta_k=0.9, rho_rot_mat=0.1, enable_gravity_prior=False, gravity_sqrt_info=10.0, ego_poses=None):
        self.split = split; self.self_id = int(split["self_id"])
        self.ids = np.asarray(split["ids"], np.int64); self.pos = {int(i): k for k, i in enumerate(self.ids)}
        self.x = np.array(split["poses"], np.float64); self.fixed = np.asarray(split["fixed"]).astype(bool)
        self.owner = np.asarray(split["owner"]); self.id_a = np.asarray(split["id_a"], np.int64); self.id_b = np.asarray(split["id_b"], np.int64)
        self.eta, self.rho = float(eta_k), float(rho_rot_mat)
        self.gravity, self.g = bool(enable_gravity_prior), float(gravity_sqrt_info)
        self.ego = None if ego_poses is None else np.asarray(ego_poses, np.float64).reshape(-1, 7)
        self.named = set(self.id_a.tolist()) | set(self.id_b.tolist())
        self.duals = {}       # (neighbour, frame id) -> [y_l (9), y_r (9)], row-major 3x3
        self.inbox = []
        self.rstate = {}      # frame id -> R_state (3x3)
        self.last = None      # the last step's system and solution

    # ---- receipt and broadcast
    def rot_receive(self, msg):
        sender, target, frames, duals, poses = msg
        for f, p in zip(np.asarray(frames, np.int64), np.asarray(poses, np.float64).reshape(-1, 7)):
            i = self.pos.get(int(f))
            if i is not None and int(self.owner[i]) == int(sender):
                self.x[i] = p
        self.inbox.append((int(sender), int(target), np.asarray(frames, np.int64), np.asarray(duals, np.float64).reshape(-1, 9)))

    def rot_messages(self):
        keys = sorted(self.duals)
        out = []
        for n in sorted({k[0] for k in keys}):
            fs = [f for m, f in keys if m == n]
            out.append((self.self_id, n, np.array(fs, np.int64), np.array([self.duals[(n, f)][0] for f in fs]).reshape(-1, 9),
                        self.x[[self.pos[f] for f in fs]].reshape(-1, 7)))
        return out

    def table(self):
        """keys in table order, y_l [K, 9], y_r [K, 9]"""
        keys = sorted(self.duals)
        return keys, np.array([self.duals[k][0] for k in keys]).reshape(-1, 9), np.array([self.duals[k][1] for k in keys]).reshape(-1, 9)

    # ---- one step
    def _process(self):
        for sender, target, frames, vals in self.inbox:
            for f, v in zip(frames, vals):
                if int(f) not in self.pos or int(f) not in self.named:
                    continue
                key = (sender, int(f))
                if target == self.self_id or key not in self.duals:
                    if key not in self.duals:
                        self.duals[key] = [v.copy(), v.copy()]
                    else:
                        self.duals[key][1] = v.copy()
        self.inbox = []

    def _scan(self):
        for f in np.concatenate([self.id_a, self.id_b]):
            o = int(self.owner[self.pos[int(f)]])
            if o != self.self_id and (o, int(f)) not in self.duals:
                self.duals[(o, int(f))] = [np.zeros(9), np.zeros(9)]

    def system(self):
        """(A, b, frames, col, build_system's dict) of the current step: the rows of build_system, then the dual priors in table
        order.  Raises ValueError on an unanchored component."""
        ego_ids = None if self.ego is None else self.ids
        s = build_system(self.ids, self.x, self.fixed, self.id_a, self.id_b, self.split["rel"], self.split["sqrt_info"], self.gravity, self.g,
                         ego_ids, self.ego)
        frames, col = s["frames"], s["col"]
        w = dual_weight(self.rho)
        rows, cols, vals, b = [], [], [], []
        r = 0
        for (n, f), (_, yr) in sorted(self.duals.items()):
            if f not in col:
                continue
            Y = yr.reshape(3, 3)
            for k in range(3):
                for j in range(3):
                    rows.append(r + 3 * k + j); cols.append(9 * col[f] + 3 * k + j); vals.append(w)
                b += list(w * Y[k])
            r += 9
        Ad = sp.csr_matrix((vals, (rows, cols)), shape=(r, 9 * len(frames)))
        self._check_anchored(s, col)
        return sp.vstack([s["A"], Ad]).tocsr(), np.concatenate([s["b"], np.array(b)]), frames, col, s

    def _check_anchored(self, s, col):
        """A^T A is singular iff a component of free frames has no fixed-frame edge row and no dual prior (the reference
        asserts, base :173).  Gravity rows anchor k = 2 only, so they do not count."""
        F = len(col)
        if F == 0:
            return
        fixed_ids = set(int(i) for i, f in zip(self.ids, self.fixed) if f)
        both = [(col[int(a)], col[int(b)]) for a, b, u in zip(self.id_a, self.id_b, s["used"]) if u and int(a) in col and int(b) in col]
        G = sp.coo_matrix((np.ones(len(both)), ([p for p, _ in both], [q for _, q in both])), shape=(F, F))
        _, lab = connected_components(G, directed=False)
        anchored = set(lab[col[int(b)]] for a, b, u in zip(self.id_a, self.id_b, s["used"]) if u and int(a) in fixed_ids)
        anchored |= set(lab[col[f]] for (_, f) in self.duals if f in col)
        for f in s["frames"]:
            if lab[col[f]] not in anchored:
                raise ValueError(f"frame {f}: its component of free frames has no fixed-frame row and no dual prior")

    def rot_init_step(self):
        self._process()
        for f in self.named:
            if f not in self.rstate:
                self.rstate[f] = quat_R(self.x[self.pos[f], 3:7])
        self._scan()
        A, b, frames, col, _ = self.system()
        F = len(frames)
        chg = []
        if F:
            H = (A.T @ A).tocsc()
            sol = spla.spsolve(H, A.T @ b)
            M = np.asarray(sol).reshape(F, 3, 3)
            for f in frames:                                       # ascending frame id
                m = M[col[f]]; S = self.rstate[f]
                with np.errstate(divide="ignore", invalid="ignore"):   # R_state = 0 after a zero M: inf, as in the reference
                    chg.append(np.linalg.norm(S - m) / np.linalg.norm(S))
                self.rstate[f] = m.copy()
                if int(self.owner[self.pos[f]]) == self.self_id:
                    self.x[self.pos[f], 3:7] = R_quat(project(m))
            self.last = dict(A=A, b=b, H=H, x=sol, frames=frames, col=col)
        else:
            self.last = dict(A=A, b=b, H=None, x=np.zeros(0), frames=frames, col=col)
        keys, yl, yr = self.table()
        if keys:
            X = np.array([self.rstate[f].ravel() for _, f in keys])
            yl = update_duals(yl, yr, X, self.eta)
            for k, key in enumerate(keys):
                self.duals[key][0] = yl[k]
        return dict(frames=F, state_changes=float(np.mean(chg)) if chg else 0.0)

    def M(self):
        """R_state per frame of the split [n, 3, 3] (0 where the frame has not entered a step)."""
        return np.array([self.rstate.get(int(f), np.zeros((3, 3))) for f in self.ids]).reshape(-1, 3, 3)


def run(agents, rounds, after_round=None):
    """The synchronous schedule: every agent steps, then every message of the round goes to every other agent.  Returns the
    per-round lists of step reports."""
    out = []
    for r in range(rounds):
        reps = [a.rot_init_step() for a in agents]
        msgs = [m for a in agents for m in a.rot_messages()]
        for a in agents:
            for m in msgs:
                if m[0] != a.self_id:
                    a.rot_receive(m)
        out.append(reps)
        if after_round is not None:
            after_round(r, agents, reps)
    return out


def kappa(agent):
    """2-norm condition number of the last step's normal matrix A^T A (dense; small graphs only)."""
    H = agent.last["H"]
    return 1.0 if H is None else float(np.linalg.cond(H.toarray()))
