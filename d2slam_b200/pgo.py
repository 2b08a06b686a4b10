"""Pose-graph side of libd2ba.so (include/d2pgo.h): ctypes binding, synthetic multi-agent pose graphs (BASELINE config 5:
10 000 poses on 8 random-walk trajectories, 40 000 edges), and g2o files in the reference's multi-agent convention.

g2o convention (d2pgo/test/posegraph_g2o.cpp:27-39, 57-232): `VERTEX_SE3:QUAT id x y z qx qy qz qw`,
`EDGE_SE3:QUAT id_a id_b x y z qx qy qz qw <21 upper-triangular information entries>`; for multi-agent files the top byte of
a vertex id carries chr('a' + agent) (gtsam Symbol style) and the low 56 bits the keyframe index.

4-DoF (d2pgo's default pgo_pose_dof = PGO_POSE_4D): `PgoSolver(pose_dof=4)` with set_poses_4d / add_edges_4d / get_poses_4d
on [x y z yaw] poses; poses_to_4d / poses_from_4d convert to and from 7-vector poses the way d2pgo does, pose_graph_to_4d
builds 4-DoF inputs from a make_pose_graph graph.

PCM (d2pgo's enable_pcm): `PgoSolver.pcm` rejects inconsistent loop closures before they are added (include/d2pgo.h
d2pgo_pcm); make_pcm_case builds its inputs from a make_pose_graph graph, with injected gross outliers.

Gravity prior (d2pgo's enable_gravity_prior, 6-DoF): `PgoSolver.add_gravity_priors` ties each pose's roll and pitch to the
gravity direction of its frame's ego (VIO) pose (include/d2pgo.h d2pgo_add_gravity_priors); make_gravity_case builds ego poses
for a make_pose_graph graph."""
import ctypes as C

import numpy as np

from .solver import lib as _lib


class PgoConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_iterations", C.c_int32), ("pcg_max_iterations", C.c_int32), ("pose_dof", C.c_int32),
                ("pcg_tolerance", C.c_double), ("lambda0", C.c_double), ("function_tolerance", C.c_double)]


class PgoReport(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("accepted", C.c_int32), ("pcg_iterations", C.c_int32), ("converged", C.c_int32),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("device_ms", C.c_double)]


class PcmConfig(C.Structure):
    _fields_ = [("pcm_thres", C.c_double), ("pos_covariance_per_meter", C.c_double), ("yaw_covariance_per_meter", C.c_double)]


class PcmReport(C.Structure):
    _fields_ = [("groups", C.c_int32), ("inliers", C.c_int32), ("pairs_tested", C.c_int64), ("consistent_pairs", C.c_int64),
                ("clique_rounds", C.c_int64), ("device_ms", C.c_double), ("pair_ms", C.c_double), ("clique_ms", C.c_double)]


PGO_EXPORTED = ["d2pgo_default_config", "d2pgo_create", "d2pgo_destroy", "d2pgo_last_error", "d2pgo_set_poses", "d2pgo_add_edges",
                "d2pgo_comm_init", "d2pgo_solve", "d2pgo_get_poses", "d2pgo_debug_edges", "d2pgo_set_poses_4d", "d2pgo_add_edges_4d",
                "d2pgo_get_poses_4d", "d2pgo_default_pcm_config", "d2pgo_pcm", "d2pgo_debug_pcm_smd", "d2pgo_debug_pcm_clique",
                "d2pgo_add_gravity_priors", "d2pgo_debug_gravity_priors"]
GRAVITY_SQRT_INFO = 10.0   # d2pgo's gravity_sqrt_info (RotInitConfig, d2pgo_config.h:13; the shipped configs)
_CREATE_ERRORS = {2: "pose_dof must be 0 or 6 (6-DoF poses) or 4 ([x y z yaw] poses)", 3: "no CUDA device (there is no CPU fallback)",
                  4: "bad device index"}


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class PgoSolver:
    def __init__(self, **kw):
        L = _lib()
        L.d2pgo_last_error.restype = C.c_char_p
        L.d2pgo_last_error.argtypes = [C.c_void_p]
        self.cfg = PgoConfig()
        L.d2pgo_default_config(C.byref(self.cfg))
        for k, v in kw.items():
            setattr(self.cfg, k, v)
        self.h = C.c_void_p()
        rc = L.d2pgo_create(C.byref(self.cfg), C.byref(self.h))
        if rc:
            raise RuntimeError(f"d2pgo_create failed rc={rc}: {_CREATE_ERRORS.get(rc, 'CUDA device required; no CPU fallback')}")
        self.n_edges = 0
        self.n_priors = 0

    def _chk(self, rc, what):
        if rc:
            raise RuntimeError(f"{what} failed rc={rc}: {_lib().d2pgo_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            _lib().d2pgo_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_poses(self, ids, poses, fixed=None):
        ids = np.ascontiguousarray(ids, np.int64); poses = np.ascontiguousarray(poses, np.float64)
        f = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        self._chk(_lib().d2pgo_set_poses(self.h, C.c_int32(len(ids)), _p(ids), _p(poses), _p(f)), "set_poses")
        self.n_edges = 0
        self.n_priors = 0

    def add_edges(self, id_a, id_b, rel, sqrt_info):
        id_a = np.ascontiguousarray(id_a, np.int64); id_b = np.ascontiguousarray(id_b, np.int64)
        rel = np.ascontiguousarray(rel, np.float64); si = np.ascontiguousarray(sqrt_info, np.float64)
        self._chk(_lib().d2pgo_add_edges(self.h, C.c_int32(len(id_a)), _p(id_a), _p(id_b), _p(rel), _p(si)), "add_edges")
        self.n_edges += len(id_a)

    def set_poses_4d(self, ids, poses4, fixed=None):
        """[x y z yaw] poses of a pose_dof = 4 solver."""
        ids = np.ascontiguousarray(ids, np.int64); poses4 = np.ascontiguousarray(poses4, np.float64)
        f = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        self._chk(_lib().d2pgo_set_poses_4d(self.h, C.c_int32(len(ids)), _p(ids), _p(poses4), _p(f)), "set_poses_4d")
        self.n_edges = 0
        self.n_priors = 0

    def add_edges_4d(self, id_a, id_b, rel4, sqrt_info16):
        """rel4 = [x y z yaw] measurements (RelPoseFactor4D), sqrt_info16 = 4x4 square-root information per edge."""
        id_a = np.ascontiguousarray(id_a, np.int64); id_b = np.ascontiguousarray(id_b, np.int64)
        rel4 = np.ascontiguousarray(rel4, np.float64); si = np.ascontiguousarray(sqrt_info16, np.float64)
        self._chk(_lib().d2pgo_add_edges_4d(self.h, C.c_int32(len(id_a)), _p(id_a), _p(id_b), _p(rel4), _p(si)), "add_edges_4d")
        self.n_edges += len(id_a)

    def add_gravity_priors(self, ids, ego_poses7, sqrt_info=None):
        """One gravity prior per id (d2pgo's setupGravityPriorFactors): r = S^T (R_i^T e3 - R_ego^T e3) with the frame's ego pose
        [x y z qx qy qz qw]; sqrt_info = [n, 3, 3] (or [n, 9]) S, None = GRAVITY_SQRT_INFO * I3 for every prior.  6-DoF only."""
        ids = np.ascontiguousarray(ids, np.int64); ego = np.ascontiguousarray(np.asarray(ego_poses7, np.float64).reshape(-1, 7))
        S = np.tile(GRAVITY_SQRT_INFO * np.eye(3), (len(ids), 1, 1)) if sqrt_info is None else np.asarray(sqrt_info, np.float64)
        S = np.ascontiguousarray(S.reshape(-1, 9))
        self._chk(_lib().d2pgo_add_gravity_priors(self.h, C.c_int32(len(ids)), _p(ids), _p(ego), _p(S)), "add_gravity_priors")
        self.n_priors += len(ids)

    def debug_gravity_priors(self):
        """Per local gravity prior at the current poses: r (3) | J (3 x 6 in the tangent [dp, dtheta]), 21 doubles."""
        out = np.zeros((max(self.n_priors, 1), 21))
        self._chk(_lib().d2pgo_debug_gravity_priors(self.h, _p(out), C.c_int64(out.size)), "debug_gravity_priors")
        return out[: self.n_priors]

    def comm_init(self, unique_id, rank, nranks):
        uid = (C.c_uint8 * 128)(*unique_id)
        self._chk(_lib().d2pgo_comm_init(self.h, uid, C.c_int32(rank), C.c_int32(nranks)), "comm_init")

    def solve(self):
        r = PgoReport()
        self._chk(_lib().d2pgo_solve(self.h, C.byref(r)), "solve")
        return r

    def get_poses(self, ids):
        ids = np.ascontiguousarray(ids, np.int64); out = np.zeros((len(ids), 7))
        self._chk(_lib().d2pgo_get_poses(self.h, C.c_int32(len(ids)), _p(ids), _p(out)), "get_poses")
        return out

    def get_poses_4d(self, ids):
        ids = np.ascontiguousarray(ids, np.int64); out = np.zeros((len(ids), 4))
        self._chk(_lib().d2pgo_get_poses_4d(self.h, C.c_int32(len(ids)), _p(ids), _p(out)), "get_poses_4d")
        return out

    def debug_edges(self):
        """Per local edge: r | J_a | J_b at the current poses, 78 doubles (6-DoF) or 36 (pose_dof = 4)."""
        out = np.zeros((max(self.n_edges, 1), 36 if self.cfg.pose_dof == 4 else 78))
        self._chk(_lib().d2pgo_debug_edges(self.h, _p(out), C.c_int64(out.size)), "debug_edges")
        return out[: self.n_edges]

    def pcm(self, frame_ids, frame_agent, ego_poses7, kf_a, kf_b, rel7, sqrt_info36, **cfg):
        """Loop-closure outlier rejection (d2pgo's enable_pcm; include/d2pgo.h d2pgo_pcm): boolean inlier mask over the loops.
        cfg overrides PcmConfig fields (pcm_thres, pos_covariance_per_meter, yaw_covariance_per_meter); the report of the
        call is kept in self.pcm_report.  The handle's poses and edges are not touched."""
        c = PcmConfig()
        _lib().d2pgo_default_pcm_config(C.byref(c))
        for k, v in cfg.items():
            setattr(c, k, v)
        fid = np.ascontiguousarray(frame_ids, np.int64); fag = np.ascontiguousarray(frame_agent, np.int32)
        ego = np.ascontiguousarray(ego_poses7, np.float64).reshape(-1, 7)
        ka = np.ascontiguousarray(kf_a, np.int64); kb = np.ascontiguousarray(kf_b, np.int64)
        rel = np.ascontiguousarray(rel7, np.float64).reshape(-1, 7); si = np.ascontiguousarray(sqrt_info36, np.float64).reshape(-1, 36)
        out = np.zeros(max(len(ka), 1), np.uint8); r = PcmReport()
        self._chk(_lib().d2pgo_pcm(self.h, C.byref(c), C.c_int32(len(fid)), _p(fid), _p(fag), _p(ego), C.c_int32(len(ka)), _p(ka), _p(kb), _p(rel), _p(si),
                                   _p(out), C.byref(r)), "pcm")
        self.pcm_report = r
        return out[: len(ka)].astype(bool)

    def debug_pcm_smd(self):
        """smd of every tested loop pair (i, j < i) of the last pcm() call, group-major (include/d2pgo.h)."""
        out = np.zeros(max(int(self.pcm_report.pairs_tested), 1))
        self._chk(_lib().d2pgo_debug_pcm_smd(self.h, _p(out), C.c_int64(out.size)), "debug_pcm_smd")
        return out[: int(self.pcm_report.pairs_tested)]

    def debug_pcm_clique(self, adj):
        """The device clique kernel alone on a symmetric boolean adjacency [n, n] -> boolean membership [n]."""
        words = pcm_pack_bits(adj)
        n = len(words); member = np.zeros(max(n, 1), np.uint8); size = C.c_int32()
        self._chk(_lib().d2pgo_debug_pcm_clique(self.h, C.c_int32(n), _p(words), _p(member), C.byref(size)), "debug_pcm_clique")
        return member[:n].astype(bool)


def pcm_pack_bits(adj):
    """Boolean [n, n] -> uint32 rows [n, ceil(n / 32)], bit j of row i = word j // 32, bit j % 32 (d2pgo_debug_pcm_clique)."""
    adj = np.asarray(adj, bool); n = len(adj); W = (n + 31) // 32
    pad = np.zeros((n, W * 32), bool); pad[:, :n] = adj
    return np.ascontiguousarray((pad.reshape(n, W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32))


# ------------------------------------------------------------------------------------------------ synthetic graphs
def _qmul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def _qconj(q):
    return q * np.array([-1.0, -1.0, -1.0, 1.0])


def _qrot(q, v):
    qv = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], axis=-1)
    return _qmul(_qmul(q, qv), _qconj(q))[..., :3]


def _qexp(th):
    a = np.linalg.norm(th, axis=-1, keepdims=True)
    s = np.where(a < 1e-12, 0.5, np.sin(a / 2) / np.where(a < 1e-12, 1.0, a))
    return np.concatenate([th * s, np.cos(a / 2)], axis=-1)


def relative_pose(pa, pb):
    """T_a^-1 T_b as [t, q]."""
    qi = _qconj(pa[..., 3:7])
    return np.concatenate([_qrot(qi, pb[..., :3] - pa[..., :3]), _qmul(qi, pb[..., 3:7])], axis=-1)


def make_pose_graph(seed=0, n_agents=8, poses_per_agent=1250, loops=30000, sigma_t=0.05, sigma_r=np.deg2rad(1.0), loop_radius=5.0):
    """Random-walk trajectories (one per agent) + odometry edges + loop closures between poses within `loop_radius`
    (SURVEY.md 8d PGO config).  ids: agent * 1_000_000 + index.  Returns dict(ids, gt, init, fixed, id_a, id_b, rel, sqrt_info, agent)."""
    rng = np.random.default_rng(seed)
    gt = []
    for a in range(n_agents):
        p = np.zeros((poses_per_agent, 7)); p[0, :3] = rng.uniform(-10, 10, 3) * np.array([1, 1, 0.2]); p[0, 3:7] = _qexp(rng.normal(0, 0.3, 3) * np.array([0.2, 0.2, 3.0]))
        steps_t = np.abs(rng.normal(0.4, 0.1, (poses_per_agent, 1))) * np.array([1.0, 0.0, 0.0]) + rng.normal(0, 0.03, (poses_per_agent, 3))
        steps_r = rng.normal(0, 0.08, (poses_per_agent, 3)) * np.array([0.2, 0.2, 1.0])
        for k in range(1, poses_per_agent):
            p[k, :3] = p[k - 1, :3] + _qrot(p[k - 1, 3:7], steps_t[k]); q = _qmul(p[k - 1, 3:7], _qexp(steps_r[k])); p[k, 3:7] = q / np.linalg.norm(q)
        gt.append(p)
    gt = np.concatenate(gt); N = len(gt)
    agent = np.repeat(np.arange(n_agents), poses_per_agent)
    ids = (agent.astype(np.int64) * 1_000_000 + np.tile(np.arange(poses_per_agent), n_agents)).astype(np.int64)
    ia = [np.arange(a * poses_per_agent, (a + 1) * poses_per_agent - 1) for a in range(n_agents)]
    ia = np.concatenate(ia); ib = ia + 1
    # loop closures: random pairs within the radius (grid hashing)
    cell = np.floor(gt[:, :2] / loop_radius).astype(np.int64); key = cell[:, 0] * 100003 + cell[:, 1]
    order = np.argsort(key); ks = key[order]
    la, lb = [], []
    tries = 0
    while len(la) < loops and tries < 50:
        i = rng.integers(0, N, loops)
        lo = np.searchsorted(ks, key[i], "left"); hi = np.searchsorted(ks, key[i], "right")
        j = order[(lo + (rng.random(loops) * (hi - lo)).astype(np.int64)).clip(0, N - 1)]
        ok = (np.abs(i - j) > 5) & (np.linalg.norm(gt[i, :3] - gt[j, :3], axis=1) < loop_radius)
        la += i[ok].tolist(); lb += j[ok].tolist(); tries += 1
    la = la[:loops]; lb = lb[:loops]
    # one guaranteed inter-agent closure per agent (closest pair to any earlier agent) so that the graph is connected and the
    # single fixed pose removes the whole gauge freedom
    for a in range(1, n_agents):
        mine = np.arange(a * poses_per_agent, (a + 1) * poses_per_agent); prev = np.arange(0, a * poses_per_agent)
        sub = prev[:: max(1, len(prev) // 2000)]
        d2 = ((gt[mine, None, :3] - gt[None, sub, :3]) ** 2).sum(-1)
        i, j = np.unravel_index(np.argmin(d2), d2.shape)
        la.append(int(mine[i])); lb.append(int(sub[j]))
    la = np.array(la, np.int64); lb = np.array(lb, np.int64)
    ea = np.concatenate([ia, la]); eb = np.concatenate([ib, lb]); E = len(ea)
    rel = relative_pose(gt[ea], gt[eb])
    rel[:, :3] += rng.normal(0, sigma_t, (E, 3))
    q = _qmul(rel[:, 3:7], _qexp(rng.normal(0, sigma_r, (E, 3)))); rel[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    si = np.zeros((E, 6, 6)); si[:, [0, 1, 2], [0, 1, 2]] = 1.0 / sigma_t; si[:, [3, 4, 5], [3, 4, 5]] = 1.0 / sigma_r
    # initial guess: odometry chained per agent (drifts), first pose of every agent from ground truth + noise
    init = gt.copy()
    for a in range(n_agents):
        s = a * poses_per_agent
        init[s, :3] += rng.normal(0, 0.2, 3)
        for k in range(1, poses_per_agent):
            r = rel[s - a + k - 1] if False else rel[(s - a) + k - 1]   # odometry edge index of (s+k-1 -> s+k)
            init[s + k, :3] = init[s + k - 1, :3] + _qrot(init[s + k - 1, 3:7], r[:3]); q = _qmul(init[s + k - 1, 3:7], r[3:7]); init[s + k, 3:7] = q / np.linalg.norm(q)
    fixed = np.zeros(N, np.uint8); fixed[0] = 1; init[0] = gt[0]
    return dict(ids=ids, gt=gt, init=init, fixed=fixed, id_a=ids[ea], id_b=ids[eb], rel=rel, sqrt_info=si.reshape(E, 36), agent=agent, ea=ea, eb=eb)


# ------------------------------------------------------------------------------------------------ 4-DoF poses
def normalize_angle(a):
    """Utility::NormalizeAngle (utils.hpp:251-257): a - 2 pi floor((a + pi) / 2 pi), in [-pi, pi)."""
    return a - 2.0 * np.pi * np.floor((a + np.pi) / (2.0 * np.pi))


def quat_yaw(q):
    """Yaw of [qx qy qz qw] quaternions: the z angle of the z-y-x Euler decomposition, atan2(2(w z + x y), 1 - 2(y^2 + z^2)).
    ASSUMED to be Swarm::Pose::yaw (swarm_msgs is not in the reference tree); the same formula pins RelPoseFactor4D's
    measurement yaw to the reference functor."""
    q = np.asarray(q, np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))


def _qyaw(yaw):
    yaw = np.asarray(yaw, np.float64)
    z = np.zeros_like(yaw)
    return np.stack([z, z, np.sin(yaw / 2), np.cos(yaw / 2)], axis=-1)


def poses_to_4d(poses7):
    """[x y z qx qy qz qw] -> [x y z yaw], as PGOState::addFrame's 4-DoF branch takes a frame (pgostate.hpp:31-33,
    Swarm::Pose::to_vector_xyzyaw; yaw by quat_yaw, the ASSUMED Swarm::Pose::yaw)."""
    p = np.asarray(poses7, np.float64)
    return np.concatenate([p[..., :3], quat_yaw(p[..., 3:7])[..., None]], axis=-1)


def poses_from_4d(x4, ego_poses7):
    """Solved [x y z yaw] -> [x y z qx qy qz qw] with the ego pose's roll and pitch put back, as D2PGO::getOptimizedTrajs does
    for 4-DoF (d2pgo.cpp:640-645): q = Rz(yaw) (yaw_only(q_ego)^-1 q_ego)."""
    x4 = np.asarray(x4, np.float64); qe = np.asarray(ego_poses7, np.float64)[..., 3:7]
    tilt = _qmul(_qconj(_qyaw(quat_yaw(qe))), qe)
    q = _qmul(_qyaw(x4[..., 3]), tilt)
    return np.concatenate([x4[..., :3], q / np.linalg.norm(q, axis=-1, keepdims=True)], axis=-1)


def pose_graph_to_4d(g, seed=0, sigma_t=0.05, sigma_yaw=np.deg2rad(1.0)):
    """4-DoF inputs from a make_pose_graph graph: the same ground truth (as [x y z yaw]) and the same edge topology, measurements
    Rz(-yaw_a)(p_b - p_a) + noise and N(yaw_b - yaw_a + noise), diagonal square-root information, initial guess chained from the
    odometry edges per agent (first pose of every agent from ground truth + noise), pose 0 fixed at ground truth.
    Returns dict(ids, gt, init, fixed, id_a, id_b, ea, eb, rel, sqrt_info, agent) with 4-vectors and [E, 16] sqrt_info."""
    rng = np.random.default_rng(seed)
    gt = poses_to_4d(g["gt"]); ea = np.asarray(g["ea"]); eb = np.asarray(g["eb"]); agent = np.asarray(g["agent"])
    E = len(ea)
    c, s = np.cos(-gt[ea, 3]), np.sin(-gt[ea, 3]); v = gt[eb, :3] - gt[ea, :3]
    rel = np.zeros((E, 4))
    rel[:, 0] = c * v[:, 0] - s * v[:, 1] + rng.normal(0, sigma_t, E)
    rel[:, 1] = s * v[:, 0] + c * v[:, 1] + rng.normal(0, sigma_t, E)
    rel[:, 2] = v[:, 2] + rng.normal(0, sigma_t, E)
    rel[:, 3] = normalize_angle(gt[eb, 3] - gt[ea, 3] + rng.normal(0, sigma_yaw, E))
    si = np.zeros((E, 4, 4)); si[:, [0, 1, 2], [0, 1, 2]] = 1.0 / sigma_t; si[:, 3, 3] = 1.0 / sigma_yaw
    # odometry edges: e -> (i, i + 1) within one agent; each pose after an agent's first has exactly one (make_pose_graph lists
    # them first)
    odo = np.full(len(gt), -1)
    n_odo = len(gt) - len(np.unique(agent))
    assert np.all(eb[:n_odo] == ea[:n_odo] + 1) and np.all(agent[ea[:n_odo]] == agent[eb[:n_odo]])
    odo[eb[:n_odo]] = np.arange(n_odo)
    init = gt.copy()
    for a in np.unique(agent):
        idx = np.nonzero(agent == a)[0]; s0 = idx[0]
        e = odo[idx[1:]]
        assert np.all(e >= 0)
        init[s0, :3] += rng.normal(0, 0.2, 3)
        yaw = init[s0, 3] + np.concatenate([[0.0], np.cumsum(rel[e, 3])])
        c, s = np.cos(yaw[:-1]), np.sin(yaw[:-1])
        step = np.stack([c * rel[e, 0] - s * rel[e, 1], s * rel[e, 0] + c * rel[e, 1], rel[e, 2]], axis=1)
        init[idx, :3] = init[s0, :3] + np.concatenate([np.zeros((1, 3)), np.cumsum(step, axis=0)])
        init[idx, 3] = normalize_angle(yaw)
    fixed = np.zeros(len(gt), np.uint8); fixed[0] = 1; init[0] = gt[0]
    return dict(ids=np.asarray(g["ids"]), gt=gt, init=init, fixed=fixed, id_a=np.asarray(g["id_a"]), id_b=np.asarray(g["id_b"]), ea=ea, eb=eb,
                rel=rel, sqrt_info=si.reshape(E, 16), agent=agent)


# ------------------------------------------------------------------------------------------------ PCM cases
def _odometry_chain(g):
    """Per-agent ego trajectories: the first pose of every agent from ground truth, then the odometry edges composed."""
    gt = np.asarray(g["gt"]); agent = np.asarray(g["agent"]); ea = np.asarray(g["ea"]); eb = np.asarray(g["eb"]); rel = np.asarray(g["rel"])
    n_odo = len(gt) - len(np.unique(agent))
    assert np.all(eb[:n_odo] == ea[:n_odo] + 1)
    ego = gt.copy()
    for e in range(n_odo):
        a, b = ea[e], eb[e]
        ego[b, :3] = ego[a, :3] + _qrot(ego[a, 3:7], rel[e, :3]); q = _qmul(ego[a, 3:7], rel[e, 3:7]); ego[b, 3:7] = q / np.linalg.norm(q)
    return ego, n_odo


def make_pcm_case(g, outlier_frac=0.05, seed=0):
    """A PCM input from a make_pose_graph graph: frames = every pose with its agent and its ego pose (the agent's odometry
    chain), loops = the edges after the odometry edges, `rel_bad` = the same loops with a fraction turned into gross
    outliers (2-10 m of translation in a random direction and 20-180 degrees of yaw, random sign), `outlier` = which,
    `bad_dt` / `bad_yaw` = the perturbations of the outliers in loop order (to corrupt 4-DoF measurements the same way)."""
    rng = np.random.default_rng(seed)
    ego, n_odo = _odometry_chain(g)
    ids = np.asarray(g["ids"]); agent = np.asarray(g["agent"]).astype(np.int32)
    rel = np.array(g["rel"][n_odo:]); L = len(rel)
    bad = np.zeros(L, bool); bad[rng.choice(L, int(round(outlier_frac * L)), replace=False)] = True
    k = int(bad.sum())
    d = rng.normal(size=(k, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rel_bad = rel.copy()
    rel_bad[bad, :3] += d * rng.uniform(2.0, 10.0, (k, 1))
    yaw = rng.uniform(np.deg2rad(20), np.pi, k) * rng.choice([-1.0, 1.0], k)
    q = _qmul(rel_bad[bad, 3:7], _qyaw(yaw)); rel_bad[bad, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return dict(frame_ids=ids, frame_agent=agent, ego=ego, kf_a=np.asarray(g["id_a"][n_odo:]), kf_b=np.asarray(g["id_b"][n_odo:]), rel=rel,
                rel_bad=rel_bad, sqrt_info=np.asarray(g["sqrt_info"][n_odo:]), outlier=bad, bad_dt=d * np.linalg.norm(rel_bad[bad, :3] - rel[bad, :3], axis=1, keepdims=True),
                bad_yaw=yaw, n_odo=n_odo)


# ------------------------------------------------------------------------------------------------ gravity priors
def make_gravity_case(g, sigma_tilt=np.deg2rad(0.5), seed=0):
    """Ego (VIO) poses for gravity priors on a make_pose_graph graph: position and yaw from the agent's odometry chain
    (_odometry_chain), roll and pitch from the ground truth turned by a random rotation of sigma_tilt per axis -- the gravity
    direction a VIO front end observes.  The graph's own odometry drifts in roll and pitch, which the priors correct.
    Returns dict(ids, ego) with ego [N, 7]."""
    rng = np.random.default_rng(seed)
    chain, _ = _odometry_chain(g)
    gt = np.asarray(g["gt"])
    tilt = _qmul(_qconj(_qyaw(quat_yaw(gt[:, 3:7]))), gt[:, 3:7])                 # ground-truth roll and pitch (zero yaw)
    tilt = _qmul(tilt, _qexp(rng.normal(0.0, sigma_tilt, (len(gt), 3))))
    q = _qmul(_qyaw(quat_yaw(chain[:, 3:7])), tilt)
    ego = np.concatenate([chain[:, :3], q / np.linalg.norm(q, axis=1, keepdims=True)], axis=1)
    return dict(ids=np.asarray(g["ids"]), ego=ego)


# ------------------------------------------------------------------------------------------------ g2o files
_IDX_AGENT_MIN = 1 << 56


def g2o_vertex_id(agent, index, multi=True):
    return (int(ord("a") + agent) << 56) | int(index) if multi else int(index)


def g2o_split_id(v):
    """posegraph_g2o.cpp:27-39 extrackKeyframeId: (agent, keyframe index)."""
    v = int(v)
    if v < _IDX_AGENT_MIN:
        return 0, v
    return ((v >> 56) & 255) - 97, v & ((1 << 56) - 1)


def write_g2o(path, ids, poses, id_a, id_b, rel, sqrt_info, multi=True):
    def vid(i):
        return g2o_vertex_id(int(i) // 1_000_000, int(i) % 1_000_000, multi)
    with open(path, "w") as f:
        for i, p in zip(ids, poses):
            f.write("VERTEX_SE3:QUAT %d %s\n" % (vid(i), " ".join(repr(float(x)) for x in p)))
        for a, b, r, s in zip(id_a, id_b, rel, np.asarray(sqrt_info).reshape(-1, 6, 6)):
            info = s.T @ s
            up = [info[i, j] for i in range(6) for j in range(i, 6)]
            f.write("EDGE_SE3:QUAT %d %d %s %s\n" % (vid(a), vid(b), " ".join(repr(float(x)) for x in r), " ".join(repr(float(x)) for x in up)))


def read_g2o(path, max_agent_id=1000):
    """-> dict(ids, poses, id_a, id_b, rel, sqrt_info); ids = agent * 1_000_000 + keyframe index (the estimator's frame-id
    convention, d2frontend_types.h:10-14).  Edges touching an agent above max_agent_id are skipped like the reference reader."""
    ids, poses, ea, eb, rel, si = [], [], [], [], [], []
    for line in open(path):
        t = line.split()
        if not t:
            continue
        if t[0] == "VERTEX_SE3:QUAT":
            ag, k = g2o_split_id(t[1])
            if ag > max_agent_id:
                continue
            p = np.array(t[2:9], float); p[3:7] /= np.linalg.norm(p[3:7])
            ids.append(ag * 1_000_000 + k); poses.append(p)
        elif t[0] == "EDGE_SE3:QUAT":
            (aa, ka), (ab, kb) = g2o_split_id(t[1]), g2o_split_id(t[2])
            if aa > max_agent_id or ab > max_agent_id:
                continue
            r = np.array(t[3:10], float); r[3:7] /= np.linalg.norm(r[3:7])
            up = np.array(t[10:31], float); info = np.zeros((6, 6)); k = 0
            for i in range(6):
                for j in range(i, 6):
                    info[i, j] = info[j, i] = up[k]; k += 1
            ea.append(aa * 1_000_000 + ka); eb.append(ab * 1_000_000 + kb); rel.append(r)
            w, V = np.linalg.eigh(info)           # symmetric square root of the information matrix
            si.append((V * np.sqrt(np.maximum(w, 0.0))) @ V.T)
    return dict(ids=np.array(ids, np.int64), poses=np.array(poses), id_a=np.array(ea, np.int64), id_b=np.array(eb, np.int64),
                rel=np.array(rel), sqrt_info=np.array(si).reshape(-1, 36))


def write_g2o_agents(directory, ids, poses, id_a, id_b, rel, sqrt_info):
    """The reference's multi-agent layout (read_g2o_multi_agents, posegraph_g2o.cpp:177-195): one file `<agent>.g2o` per
    agent with that agent's vertices and the edges that start at one of them (inter-agent edges name the other agent through the
    agent byte of the vertex id)."""
    import os
    ids = np.asarray(ids); id_a = np.asarray(id_a)
    agents = sorted(set(int(i) // 1_000_000 for i in ids))
    for a in agents:
        v = (ids // 1_000_000) == a; e = (id_a // 1_000_000) == a
        write_g2o(os.path.join(directory, f"{a}.g2o"), ids[v], np.asarray(poses)[v], id_a[e], np.asarray(id_b)[e], np.asarray(rel)[e], np.asarray(sqrt_info).reshape(-1, 36)[e])
    return agents


def read_g2o_agents(directory, agents_num):
    """Mirror of read_g2o_multi_agents: the numerically named *.g2o files in ascending order, the first `agents_num` of them,
    vertices / edges of agents above agents_num - 1 dropped; concatenated into one graph."""
    import os
    files = sorted((int(f[:-4]), os.path.join(directory, f)) for f in os.listdir(directory) if f.endswith(".g2o") and f[:-4].isdigit())[:agents_num]
    parts = [read_g2o(p, max_agent_id=agents_num - 1) for _, p in files]
    cat = lambda k: np.concatenate([q[k] for q in parts]) if parts else np.zeros(0)
    return dict(ids=cat("ids"), poses=cat("poses"), id_a=cat("id_a"), id_b=cat("id_b"), rel=cat("rel"), sqrt_info=cat("sqrt_info"))
