"""numpy / scipy restatement of d2pgo's chordal rotation initialisation (RotationInitialization<double>::solve,
d2pgo/src/rot_init/rotation_initialization_base.hpp; the non-distributed RotInit path of rotation_initialization.cpp:21-28),
solved sparse-direct.  Checks include/d2pgo.h d2pgo_rot_init.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_rotinit.py and tools/pgo_rotinit_bench.py.  Nothing under d2slam_b200/ imports
it.  Line numbers below are those of rotation_initialization_base.hpp unless stated.

ASSUMED: Swarm::PosePrior (swarm_msgs, not in the reference tree) built from a loop's information matrix returns that loop's
rotation square-root block from getSqrtInfoMatRot(), so the prior of an edge from a fixed frame has the edge's weight s.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.sparse.csgraph import connected_components


def quat_R(q):
    """Rotation matrices of [.., 4] xyzw quaternions, normalised first (Swarm::Pose normalises its attitude; Eigen's
    toRotationMatrix polynomial)."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def R_quat(R):
    """Eigen's Quaternion(Matrix3) (trace branch, else the largest diagonal's), xyzw, [.., 3, 3] -> [.., 4]."""
    R = np.asarray(R, np.float64)
    out = np.zeros(R.shape[:-2] + (4,))
    for idx in np.ndindex(R.shape[:-2]):
        m = R[idx]; q = np.zeros(4)
        t = np.trace(m)
        if t > 0:
            t = np.sqrt(t + 1.0); q[3] = 0.5 * t; t = 0.5 / t
            q[0] = (m[2, 1] - m[1, 2]) * t; q[1] = (m[0, 2] - m[2, 0]) * t; q[2] = (m[1, 0] - m[0, 1]) * t
        else:
            i = 0
            if m[1, 1] > m[0, 0]:
                i = 1
            if m[2, 2] > m[i, i]:
                i = 2
            j = (i + 1) % 3; k = (j + 1) % 3
            t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0); q[i] = 0.5 * t; t = 0.5 / t
            q[3] = (m[k, j] - m[j, k]) * t; q[j] = (m[j, i] + m[i, j]) * t; q[k] = (m[k, i] + m[i, k]) * t
        out[idx] = q
    return out


def project_so3(M):
    """Utility::recoverRotationSVD (d2common/include/d2common/utils.hpp:121-129): U diag(1, 1, det(U V^T)) V^T, singular values
    descending, [.., 3, 3]."""
    U, _, Vt = np.linalg.svd(M)
    d = np.linalg.det(U @ Vt)
    D = np.zeros(M.shape); D[..., 0, 0] = 1.0; D[..., 1, 1] = 1.0; D[..., 2, 2] = d
    return U @ D @ Vt


def build_system(ids, poses, fixed, id_a, id_b, rel, sqrt_info, gravity=False, gravity_sqrt_info=10.0, ego_ids=None, ego_poses=None):
    """The sparse least-squares system A x = b of solveLinearRot (:178-213).  Returns dict(A, b, frames (free frame ids,
    ascending: updateFrameIdx :57-69 over the std::set all_frames of :444-450), col (frame id -> unknown index), used, dropped).
    x[9 idx + 3 k + j] = R_f[k, j] (rows of R_f, :372)."""
    ids = np.asarray(ids, np.int64); poses = np.asarray(poses, np.float64); fixed = np.asarray(fixed).astype(bool)
    id_a = np.asarray(id_a, np.int64); id_b = np.asarray(id_b, np.int64)
    rel = np.asarray(rel, np.float64).reshape(-1, 7); S = np.asarray(sqrt_info, np.float64).reshape(-1, 6, 6)
    pos = {int(i): k for k, i in enumerate(ids)}
    is_fixed = {int(i): bool(fixed[k]) for k, i in enumerate(ids)}
    all_frames = sorted(set(id_a.tolist()) | set(id_b.tolist()))                     # :444-450
    frames = [f for f in all_frames if not is_fixed[f]]                              # :57-69
    col = {f: k for k, f in enumerate(frames)}
    rows, cols, vals, b = [], [], [], []
    row = 0
    Rrel = quat_R(rel[:, 3:7])
    s_rot = np.linalg.norm(S[:, 3:6, 3:6], axis=(1, 2))                               # sqrt_info.norm() (:103, :122)
    used = np.zeros(len(id_a), bool)

    def put(r0, c0, M):
        for i in range(3):
            for j in range(3):
                rows.append(r0 + i); cols.append(c0 + j); vals.append(M[i, j])

    for e in range(len(id_a)):                                                       # setupRotInitProblembyLoop (:89-111)
        a, bb = int(id_a[e]), int(id_b[e])
        ia, ib = col.get(a, -1), col.get(bb, -1)
        if ia == ib or ia == -1 or ib == -1:
            continue
        used[e] = True
        for k in range(3):
            put(row + 3 * k, 9 * ia + 3 * k, s_rot[e] * Rrel[e].T)
            put(row + 3 * k, 9 * ib + 3 * k, -s_rot[e] * np.eye(3))
        b += [0.0] * 9; row += 9
    for e in range(len(id_a)):                  # setPriorFactorsbyFixedParam (:72-87) + setupRotInitProblembyPrior (:113-129)
        a, bb = int(id_a[e]), int(id_b[e])
        if is_fixed[a] and not is_fixed[bb]:
            Rp = quat_R(poses[pos[a], 3:7]) @ Rrel[e]                                 # pose_fixed * loop.relative_pose
            target = bb
        elif not is_fixed[a] and is_fixed[bb]:
            continue                            # :84 builds the prior on frame_id_b -- the fixed frame: no unknowns (:116-118)
        else:
            continue
        used[e] = True
        ib = col[target]
        for k in range(3):
            put(row + 3 * k, 9 * ib + 3 * k, s_rot[e] * np.eye(3))
            b += list(s_rot[e] * Rp.T[:, k])                                           # sqrt_R * Rt.col(k)
        row += 9
    if gravity:                                                                      # setupRotInitProblembyGravityPrior (:131-144)
        ego = {int(i): np.asarray(p, np.float64) for i, p in zip(np.asarray(ego_ids, np.int64), np.asarray(ego_poses).reshape(-1, 7))}
        for f in frames:
            if f not in ego:
                raise ValueError(f"frame {f}: gravity rows need its ego pose")
            u = quat_R(ego[f][3:7]).T @ np.array([0.0, 0.0, 1.0])                     # att_odom.inverse() * gravity_direction
            put(row, 9 * col[f] + 6, gravity_sqrt_info * np.eye(3))
            b += list(gravity_sqrt_info * u); row += 3
    A = sp.csr_matrix((vals, (rows, cols)), shape=(row, 9 * len(frames)))
    return dict(A=A, b=np.array(b), frames=frames, col=col, used=used, dropped=int((~used).sum()))


def check_anchored(sys_, id_a, id_b, fixed_ids):
    """A^T A is singular iff some component of free frames (joined by the rows of edges with both ends free) has no prior
    row; the reference asserts there (solveLinear :156-173).  Raises ValueError naming such a frame."""
    frames, col = sys_["frames"], sys_["col"]
    F = len(frames)
    if F == 0:
        return
    ea, eb, used = np.asarray(id_a), np.asarray(id_b), sys_["used"]
    both = [(col[int(a)], col[int(b)]) for a, b, u in zip(ea, eb, used) if u and int(a) in col and int(b) in col]
    G = sp.coo_matrix((np.ones(len(both)), ([p for p, _ in both], [q for _, q in both])), shape=(F, F))
    _, lab = connected_components(G, directed=False)
    anchored = set(lab[col[int(b)]] for a, b, u in zip(ea, eb, used) if u and int(a) in fixed_ids)
    for f in frames:
        if lab[col[f]] not in anchored:
            raise ValueError(f"frame {f}: its component of free frames holds no fixed frame")


def rot_init(ids, poses, fixed, id_a, id_b, rel, sqrt_info, gravity=False, gravity_sqrt_info=10.0, ego_ids=None, ego_poses=None):
    """RotationInitialization::solve (:440-456): the system, x = (A^T A)^-1 A^T b sparse-direct (SimplicialLLT in the reference,
    solveLinear :146-176), M_f, R_f = project_so3(M_f), the quaternion (recoverRotationLLT :360-389) and the report's
    state_changes = mean over free frames of |R_before - M_f|_F / |R_before|_F (:376-388).  Returns dict(frames, M [F,3,3],
    R [F,3,3], poses (the handle's poses with the solved attitudes; positions untouched), state_changes, used, dropped, A, b, x)."""
    ids = np.asarray(ids, np.int64); poses = np.asarray(poses, np.float64)
    s = build_system(ids, poses, fixed, id_a, id_b, rel, sqrt_info, gravity, gravity_sqrt_info, ego_ids, ego_poses)
    fixed_ids = set(int(i) for i, f in zip(ids, np.asarray(fixed)) if f)
    check_anchored(s, id_a, id_b, fixed_ids)
    A, b = s["A"], s["b"]
    F = len(s["frames"])
    out = poses.copy()
    if F == 0:
        return dict(frames=[], M=np.zeros((0, 3, 3)), R=np.zeros((0, 3, 3)), poses=out, state_changes=float("nan"), used=s["used"],
                    dropped=s["dropped"], A=A, b=b, x=np.zeros(0))
    H = (A.T @ A).tocsc()
    x = spla.spsolve(H, A.T @ b)
    M = x.reshape(F, 3, 3)
    R = project_so3(M)
    pos = {int(i): k for k, i in enumerate(ids)}
    rows = np.array([pos[f] for f in s["frames"]])
    R0 = quat_R(poses[rows, 3:7])
    chg = np.linalg.norm(R0 - M, axis=(1, 2)) / np.linalg.norm(R0, axis=(1, 2))
    out[rows, 3:7] = R_quat(R)
    return dict(frames=s["frames"], M=M, R=R, poses=out, state_changes=float(chg.mean()), used=s["used"], dropped=s["dropped"], A=A, b=b, x=x)
