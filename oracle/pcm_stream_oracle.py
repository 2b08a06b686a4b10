"""CPU oracle of PCM as a stream (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

A numpy restatement of SwarmLocalOutlierRejection kept across OutlierRejectionLoopEdges calls (redundant = true;
d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:46-303), with either clique: FMC::maxCliqueHeu
(incremental_pcm = false, oracle/pcm_oracle.py fmc_heu) or FMC::maxCliqueHeuIncremental's search
(d2pgo/third_party/fast_max-clique_finder/src/findCliqueHeuInc.cpp:32-96).  The consistency test is oracle/pcm_oracle.py's.
Pinned to the reference's own code by tests/test_pgo_pcm_stream.py (live through oracle/_ref/libd2ref_pcm_stream.so, and
through tests/golden/ref_pcm_stream.npz)."""
import numpy as np

from oracle.pcm_oracle import adjacency, fmc_heu, group_smd


def fmc_heu_inc(adj, num_new, prev):
    """FMC::maxCliqueHeuIncremental's search on bitsets: m = prev; every seed s among the last num_new vertices with
    deg(s) >= m runs fmc_heu's greedy under m; a clique larger than m becomes the best one.  -> (FMC's return value
    max(prev, best size), the best clique as [s, picks...] or [] when no seed beat prev).  The reference returns its candidate
    buffer v_i_S instead of the clique (:92-94); that buffer is not restated."""
    adj = np.asarray(adj, bool); n = len(adj)
    rows = [int("".join("1" if b else "0" for b in r[::-1]) or "0", 2) for r in adj]
    deg = adj.sum(1)
    m, best = int(prev), []
    ok = sum(1 << int(u) for u in np.nonzero(deg >= m)[0])
    for s in range(n - num_new, n):
        if m > deg[s]:
            continue
        C = rows[s] & ok
        clique = [s]
        while C:
            v = C.bit_length() - 1
            clique.append(v); C &= rows[v]
        if len(clique) > m:
            m, best = len(clique), clique
            ok = sum(1 << int(u) for u in np.nonzero(deg >= m)[0])
    return m, best


class PcmStream:
    """SwarmLocalOutlierRejection kept across calls: keyframes are appended to their drone's trajectory; a loop is tested
    only the first time its id appears, against every earlier loop of its group; groups that got new loops run the clique
    again -- maxCliqueHeu (incremental = 0) or the incremental search with m = the group's set size, whose clique replaces the
    set when it beats m (incremental = 1; the set is the clique found, see fmc_heu_inc).  call() -> (inlier mask over the
    call's loops, {(max drone, min drone): smd of the pairs tested in this call, new rows i in arrival order, j < i
    ascending})."""

    def __init__(self, is_4dof, thres=1.635, pos_cov=4e-3, yaw_cov=4e-5, incremental=0):
        self.is4, self.thres, self.pos_cov, self.yaw_cov, self.inc = is_4dof, thres, pos_cov, yaw_cov, incremental
        self.frame_ids, self.frame_agent, self.ego = [], [], []
        self.fidx = {}
        self.loop = {}                            # id -> (group key, row)
        self.rows = {}                            # group key -> [(kf_a, kf_b, rel7, sqrt_info36)] in arrival order
        self.smd = {}                             # group key -> every pair's smd, rows ascending
        self.members = {}                         # group key -> sorted rows of its set

    def call(self, frame_ids, frame_agent, ego, loop_ids, kf_a, kf_b, rel7, sqrt_info36):
        for f, a, p in zip(np.asarray(frame_ids).tolist(), np.asarray(frame_agent).tolist(), np.asarray(ego, float).reshape(-1, 7)):
            if f in self.fidx:
                assert self.frame_agent[self.fidx[f]] == a
                continue
            self.fidx[f] = len(self.frame_ids); self.frame_ids.append(f); self.frame_agent.append(a); self.ego.append(p)
        rel7 = np.asarray(rel7, float).reshape(-1, 7); si = np.asarray(sqrt_info36, float).reshape(-1, 36)
        new = {}
        for e, lid in enumerate(np.asarray(loop_ids).tolist()):
            if lid in self.loop:
                continue
            x, y = self.frame_agent[self.fidx[int(kf_a[e])]], self.frame_agent[self.fidx[int(kf_b[e])]]
            key = (max(x, y), min(x, y))
            rows = self.rows.setdefault(key, [])
            self.loop[lid] = (key, len(rows)); rows.append((int(kf_a[e]), int(kf_b[e]), rel7[e], si[e]))
            new[key] = new.get(key, 0) + 1
        case = dict(frame_ids=np.array(self.frame_ids, np.int64), frame_agent=np.array(self.frame_agent), ego=np.array(self.ego).reshape(-1, 7))
        out = {}
        for key, k in new.items():
            rows = self.rows[key]; L = len(rows); L0 = L - k
            g = dict(case, kf_a=np.array([r[0] for r in rows]), kf_b=np.array([r[1] for r in rows]), rel=np.array([r[2] for r in rows]),
                     sqrt_info=np.array([r[3] for r in rows]))
            smd = group_smd(g, np.arange(L), self.is4, self.pos_cov, self.yaw_cov)
            old = self.smd.get(key, np.zeros(0))
            assert np.array_equal(smd[: len(old)], old)   # earlier pairs do not change as frames are appended
            self.smd[key] = smd; out[key] = smd[len(old):]
            A = adjacency(smd, L, self.thres)
            if self.inc:
                _, best = fmc_heu_inc(A, L - L0, len(self.members.get(key, [])))
                if best:
                    self.members[key] = sorted(best)
            else:
                self.members[key] = sorted(fmc_heu(A))
        mask = np.array([self.loop[lid][1] in self.members[self.loop[lid][0]] for lid in np.asarray(loop_ids).tolist()], bool)
        return mask, out
