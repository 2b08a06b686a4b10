"""CPU oracle of loop-closure PCM (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

A numpy restatement of SwarmLocalOutlierRejection::OutlierRejectionLoopEdges with redundant = true, incremental_pcm = false
(d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:46-303) and of FMC::maxCliqueHeu
(d2pgo/third_party/fast_max-clique_finder/src/findCliqueHeu.cpp:124-243) on bitsets.  Pinned to the reference's own code by
tests/test_pgo_pcm.py (live through oracle/_ref/libd2ref_pcm.so, and through tests/golden/ref_pcm.npz).  The ASSUMED swarm_msgs semantics are
those listed in include/d2pgo.h (d2pgo_pcm) and in oracle/_shim/swarm_msgs/drone_trajectory.hpp."""
import numpy as np

from d2slam_b200.pgo import _qconj, _qmul, _qrot, quat_yaw


def groups(agent_a, agent_b):
    """Loop indices per unordered drone pair: groups in order of their first loop, loops in input order."""
    order, idx = {}, []
    for e, (x, y) in enumerate(zip(np.asarray(agent_a).tolist(), np.asarray(agent_b).tolist())):
        k = (min(x, y), max(x, y))
        if k not in order:
            order[k] = len(idx); idx.append([])
        idx[order[k]].append(e)
    return [np.array(v, np.int64) for v in idx]


def _normalized(q):
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _mul(a, b):   # Swarm::Pose a * b, attitude normalised
    return np.concatenate([_qrot(a[:, 3:7], b[:, :3]) + a[:, :3], _normalized(_qmul(a[:, 3:7], b[:, 3:7]))], axis=1)


def _inv(a):
    qi = _qconj(a[:, 3:7])
    return np.concatenate([-_qrot(qi, a[:, :3]), qi], axis=1)


def _delta(a, b, is_4dof):
    """DeltaPose(a, b[, yaw only]) (ASSUMED yaw-only form: (Rz(-yaw_a)(p_b - p_a), Rz(yaw_b - yaw_a)))."""
    if not is_4dof:
        return _mul(_inv(a), b)
    ya = quat_yaw(a[:, 3:7]); dy = quat_yaw(b[:, 3:7]) - ya
    c, s = np.cos(ya), np.sin(ya); d = b[:, :3] - a[:, :3]
    t = np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], d[:, 2]], axis=1)
    z = np.zeros_like(dy)
    return np.concatenate([t, np.stack([z, z, np.sin(dy / 2), np.cos(dy / 2)], axis=1)], axis=1)


def log_map(p):
    """[t ; rotation vector] with angle 2 atan2(|v|, |w|), the sign of w (ASSUMED Pose::log_map = tangentSpace)."""
    v = p[:, 3:6]; w = p[:, 6]; n = np.linalg.norm(v, axis=1)
    k = np.where(n > 0, 2.0 * np.arctan2(n, np.abs(w)) * np.where(w < 0, -1.0, 1.0) / np.where(n > 0, n, 1.0), 0.0)
    return np.concatenate([p[:, :3], v * k[:, None]], axis=1)


def path_lengths(frame_agent, ego):
    """Path length of every frame from its drone's first keyframe, along the drone's keyframes in the order given."""
    frame_agent = np.asarray(frame_agent); ego = np.asarray(ego, float)
    out = np.zeros(len(ego))
    for a in np.unique(frame_agent):
        f = np.nonzero(frame_agent == a)[0]
        seg = np.linalg.norm(np.diff(ego[f, :3], axis=0), axis=1)
        out[f] = np.concatenate([[0.0], np.cumsum(seg)])
    return out


def group_smd(case, idx, is_4dof, pos_cov=4e-3, yaw_cov=4e-5, rel_key="rel"):
    """smd of every pair (i, j < i) of one group (rows i ascending, j ascending), edge1 = loop i, edge2 = loop j."""
    fidx = {int(f): k for k, f in enumerate(np.asarray(case["frame_ids"]).tolist())}
    agent = np.asarray(case["frame_agent"]); ego = np.asarray(case["ego"], float)
    ego = np.concatenate([ego[:, :3], _normalized(ego[:, 3:7])], axis=1)
    path = case.get("_path")
    if path is None:
        path = path_lengths(agent, ego)
    fa = np.array([fidx[int(k)] for k in np.asarray(case["kf_a"])[idx]]); fb = np.array([fidx[int(k)] for k in np.asarray(case["kf_b"])[idx]])
    rel = np.asarray(case[rel_key], float)[idx]; rel = np.concatenate([rel[:, :3], _normalized(rel[:, 3:7])], axis=1)
    S = np.asarray(case["sqrt_info"], float)[idx].reshape(-1, 6, 6)
    cov = np.linalg.inv(np.einsum("eki,ekj->eij", S, S))
    I, J = np.tril_indices(len(idx), -1)
    flip = agent[fa] > agent[fb]
    same = flip[I] == flip[J]
    p2 = np.where(same[:, None], rel[J], _inv(rel[J]))
    oa_to = np.where(same, fa[J], fb[J]); ob_to = np.where(same, fb[J], fa[J])

    def odom(f, g):
        ln = np.abs(path[g] - path[f])
        return _delta(ego[f], ego[g], is_4dof), pos_cov * ln + 0.5 * yaw_cov * ln * ln, yaw_cov * ln
    oa, ca_p, ca_r = odom(fa[I], oa_to)
    ob, cb_p, cb_r = odom(fb[I], ob_to)
    err = _mul(_mul(_mul(oa, p2), _inv(ob)), _inv(rel[I]))
    v = log_map(err)
    Sig = cov[I] + cov[J]
    d = np.concatenate([np.repeat((ca_p + cb_p)[:, None], 3, 1), np.repeat((ca_r + cb_r)[:, None], 3, 1)], axis=1)
    Sig[:, np.arange(6), np.arange(6)] += d
    return np.einsum("pi,pi->p", v, np.linalg.solve(Sig, v[..., None])[..., 0]) if len(I) else np.zeros(0)


def adjacency(smd, L, thres):
    """Consistency graph of one group from its pair list: consistent iff smd < (float) thres."""
    thr = float(np.float32(thres))
    A = np.zeros((L, L), bool)
    I, J = np.tril_indices(L, -1)
    ok = smd < thr
    A[I[ok], J[ok]] = True; A[J[ok], I[ok]] = True
    return A


def fmc_heu(adj, pruned=True):
    """FMC::maxCliqueHeu on a symmetric boolean adjacency, restated on bitsets: m = -1; every seed s with deg(s) >= m:
    C = N(s) & {u : deg(u) >= m}; repeat v = max C, C &= N(v); the clique {s} + picks becomes the best one when larger than
    m.  -> the clique as [s, picks...].  pruned = False drops both degree prunings (the plain greedy, for comparison)."""
    adj = np.asarray(adj, bool); n = len(adj)
    rows = [int("".join("1" if b else "0" for b in r[::-1]) or "0", 2) for r in adj]
    deg = adj.sum(1)
    m, best = -1, []
    ok = (1 << n) - 1
    for s in range(n):
        if pruned and m > deg[s]:
            continue
        C = rows[s] & ok
        clique = [s]
        while C:
            v = C.bit_length() - 1
            clique.append(v); C &= rows[v]
        if len(clique) > m:
            m, best = len(clique), clique
            if pruned:
                ok = sum(1 << int(u) for u in np.nonzero(deg >= m)[0])
    return best


def pcm(case, is_4dof, thres=1.635, pos_cov=4e-3, yaw_cov=4e-5, rel_key="rel"):
    """-> (inlier mask over the loops, smd of every tested pair, group-major)."""
    fidx = {int(f): k for k, f in enumerate(np.asarray(case["frame_ids"]).tolist())}
    agent = np.asarray(case["frame_agent"])
    aa = agent[[fidx[int(k)] for k in np.asarray(case["kf_a"])]]; ab = agent[[fidx[int(k)] for k in np.asarray(case["kf_b"])]]
    case = dict(case); case["_path"] = path_lengths(agent, np.asarray(case["ego"], float))
    good = np.zeros(len(aa), bool); smds = []
    for idx in groups(aa, ab):
        smd = group_smd(case, idx, is_4dof, pos_cov, yaw_cov, rel_key)
        smds.append(smd)
        good[idx[fmc_heu(adjacency(smd, len(idx), thres))]] = True
    return good, (np.concatenate(smds) if smds else np.zeros(0))
