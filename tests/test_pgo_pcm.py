"""PCM loop-closure outlier rejection (include/d2pgo.h d2pgo_pcm): the numpy oracle (oracle/pcm_oracle.py) pinned to the
reference's own SwarmLocalOutlierRejection and FMC code (live through oracle/_ref where the reference tree exists, and through
tests/golden/ref_pcm.npz everywhere), and the device against both."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pcm_oracle as po
from oracle import pgo4d_oracle as p4
from oracle import ref_pcm as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_pcm.npz")
LIVE = pytest.mark.skipif(not ref.available(), reason="reference PCM library not built")

# (is_4dof, pcm_thres, pos_covariance_per_meter, yaw_covariance_per_meter): the reference defaults, and rates consistent
# with make_pose_graph's noise at a threshold d2pgo's configs use
PCM_CONFIGS = {"d6_default": (0, 1.635, 4e-3, 4e-5), "d6_wide": (0, 3.5, 0.5, 1e-2), "d4_default": (1, 1.635, 4e-3, 4e-5), "d4_wide": (1, 3.5, 0.5, 1e-2)}


def small_case():
    """3 drones + one with a single loop (a one-loop group); intra- and inter-drone groups, both loop orientations, 10 %
    gross outliers."""
    g = pgo.make_pose_graph(seed=11, n_agents=4, poses_per_agent=60, loops=240, loop_radius=30.0)
    c = pgo.make_pcm_case(g, 0.1, seed=4)
    agent = np.asarray(c["frame_agent"]); fidx = {int(f): k for k, f in enumerate(c["frame_ids"])}
    aa = agent[[fidx[int(k)] for k in c["kf_a"]]]; ab = agent[[fidx[int(k)] for k in c["kf_b"]]]
    touches3 = np.nonzero((aa == 3) | (ab == 3))[0]
    keep = np.ones(len(aa), bool); keep[touches3[1:]] = False
    out = {k: (v[keep] if k in ("kf_a", "kf_b", "rel", "rel_bad", "sqrt_info", "outlier") else v) for k, v in c.items() if k not in ("bad_dt", "bad_yaw", "n_odo")}
    # inter-drone loops (the random walks rarely meet): drones 0-1 and 1-2, either orientation, from ground truth + noise,
    # every 5th one a gross outlier
    rng = np.random.default_rng(12)
    ids, gt = np.asarray(g["ids"]), np.asarray(g["gt"])
    a = np.concatenate([rng.integers(0, 60, 40), rng.integers(60, 120, 20)]); b = np.concatenate([rng.integers(60, 120, 40), rng.integers(120, 180, 20)])
    sw = rng.random(60) < 0.5
    a, b = np.where(sw, b, a), np.where(sw, a, b)
    rel = pgo.relative_pose(gt[a], gt[b]); rel[:, :3] += rng.normal(0, 0.05, (60, 3))
    bad = rel.copy(); bad[::5, :3] += rng.uniform(3, 8, (12, 3))
    out["kf_a"] = np.concatenate([out["kf_a"], ids[a]]); out["kf_b"] = np.concatenate([out["kf_b"], ids[b]])
    out["rel"] = np.concatenate([out["rel"], rel]); out["rel_bad"] = np.concatenate([out["rel_bad"], bad])
    out["sqrt_info"] = np.concatenate([out["sqrt_info"], np.tile(out["sqrt_info"][0], (60, 1))])
    out["outlier"] = np.concatenate([out["outlier"], np.arange(60) % 5 == 0])
    return out


def _group_agents(case):
    agent = np.asarray(case["frame_agent"]); fidx = {int(f): k for k, f in enumerate(np.asarray(case["frame_ids"]).tolist())}
    return agent[[fidx[int(k)] for k in case["kf_a"]]], agent[[fidx[int(k)] for k in case["kf_b"]]]


def ref_order_to_group_major(case, smd):
    """The reference computes groups in std::map order of (max drone id, min drone id); the device and the oracle list them
    in order of their first loop."""
    aa, ab = _group_agents(case)
    gr = po.groups(aa, ab)
    keys = [(max(aa[i[0]], ab[i[0]]), min(aa[i[0]], ab[i[0]])) for i in gr]
    sizes = [len(i) * (len(i) - 1) // 2 for i in gr]
    order = sorted(range(len(gr)), key=lambda k: keys[k])
    off = np.cumsum([0] + [sizes[k] for k in order]); part = {}
    for r, k in enumerate(order):
        part[k] = smd[off[r]:off[r + 1]]
    return np.concatenate([part[k] for k in range(len(gr))]) if gr else np.zeros(0)


def fmc_graphs(n_graphs=240, seed=0):
    """Seeded random graphs: planted cliques, ties, isolated vertices, plus graphs on which the unpruned greedy differs."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_graphs):
        n = int(rng.integers(1, 48))
        A = rng.random((n, n)) < rng.uniform(0.05, 0.7)
        A = np.triu(A, 1); A = A | A.T
        if k % 3 == 0 and n > 4:    # planted clique
            c = rng.choice(n, int(rng.integers(3, max(4, n // 2))), replace=False)
            A[np.ix_(c, c)] = True
        if k % 4 == 1 and n > 2:    # isolated vertices
            iso = rng.choice(n, int(rng.integers(1, n)), replace=False)
            A[iso, :] = False; A[:, iso] = False
        if k % 5 == 2 and n > 6:    # ties: disjoint cliques of one size
            A[:] = False
            for blk in np.array_split(rng.permutation(n), 3):
                A[np.ix_(blk, blk)] = True
        np.fill_diagonal(A, False)
        out.append(A)
    return out


def _gold():
    return np.load(GOLD)


def _gold_case():
    z = _gold()
    return {k[5:]: z[k] for k in z.files if k.startswith("case_")}


def _gold_graphs():
    z = _gold()
    ns, adj, sizes, cl = z["fmc_n"], z["fmc_adj"], z["fmc_size"], z["fmc_clique"]
    gs, cs, o, c = [], [], 0, 0
    for n, s in zip(ns, sizes):
        gs.append(adj[o:o + n * n].reshape(n, n)); o += n * n
        cs.append(cl[c:c + s].tolist()); c += s
    return gs, cs


# ----------------------------------------------------------------------------------------------- CPU
def test_golden_case_is_the_test_case():
    case, g = small_case(), _gold_case()
    for k in ("frame_ids", "frame_agent", "ego", "kf_a", "kf_b", "rel_bad", "sqrt_info"):
        assert np.array_equal(case[k], g[k]), k


def test_small_case_covers_every_kind_of_group():
    case = small_case()
    aa, ab = _group_agents(case)
    gr = po.groups(aa, ab)
    sizes = [len(i) for i in gr]
    assert 1 in sizes
    assert any(aa[i[0]] == ab[i[0]] for i in gr) and any(aa[i[0]] != ab[i[0]] for i in gr)
    inter = [i for i in gr if aa[i[0]] != ab[i[0]] and len(i) > 1]
    assert any(len(set((aa[i] > ab[i]).tolist())) == 2 for i in inter)   # same_robot_pair 1 and 2 both occur


@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_oracle_matches_golden_reference_pcm(name):
    is4, thr, pc, yc = PCM_CONFIGS[name]
    z = _gold(); case = _gold_case()
    good, smd = po.pcm(case, is4, thr, pc, yc, rel_key="rel_bad")
    want = z[f"{name}_smd"]
    assert smd.shape == want.shape
    assert np.all(np.abs(smd - want) <= 1e-10 * np.abs(want))
    assert np.array_equal(good, z[f"{name}_good"])


@LIVE
@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_oracle_matches_live_reference_pcm(name):
    is4, thr, pc, yc = PCM_CONFIGS[name]
    case = small_case()
    good_r, smd_r = ref.pcm(case, is4, thr, pc, yc, rel_key="rel_bad")
    good, smd = po.pcm(case, is4, thr, pc, yc, rel_key="rel_bad")
    want = ref_order_to_group_major(case, smd_r)
    assert np.all(np.abs(smd - want) <= 1e-10 * np.abs(want))
    assert np.array_equal(good, good_r)


def test_oracle_clique_equals_golden_fmc():
    gs, cs = _gold_graphs()
    assert len(gs) >= 200
    differs = 0
    for A, want in zip(gs, cs):
        got = po.fmc_heu(A)
        assert sorted(got) == want
        differs += sorted(po.fmc_heu(A, pruned=False)) != want
    assert differs >= 1   # the set holds graphs on which the unpruned greedy picks another clique


@LIVE
def test_oracle_clique_equals_live_fmc():
    for A in fmc_graphs():
        assert po.fmc_heu(A) == ref.fmc_heu(A)   # same clique, listed in the same order


def test_oracle_rejects_every_injected_outlier():
    g = pgo.make_pose_graph(seed=5, n_agents=3, poses_per_agent=200, loops=500)
    c = pgo.make_pcm_case(g, 0.05, seed=2)
    for is4 in (0, 1):
        good, _ = po.pcm(c, is4, 3.5, 0.5, 1e-2, rel_key="rel_bad")
        kept = (good & ~c["outlier"]).sum() / (~c["outlier"]).sum()
        print(f"is_4dof={is4}: inliers kept {kept:.3f}, outliers kept {(good & c['outlier']).sum()} of {c['outlier'].sum()}")
        assert not (good & c["outlier"]).any()
        assert kept > 0.85


def test_pcm_structs_layout():
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "d2pgo.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(d2pgo_pcm_config), '
            'offsetof(d2pgo_pcm_config, yaw_covariance_per_meter), sizeof(d2pgo_pcm_report), offsetof(d2pgo_pcm_report, pairs_tested), '
            'offsetof(d2pgo_pcm_report, clique_rounds), offsetof(d2pgo_pcm_report, clique_ms));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe]).decode().split()))
    assert out == [C.sizeof(pgo.PcmConfig), pgo.PcmConfig.yaw_covariance_per_meter.offset, C.sizeof(pgo.PcmReport), pgo.PcmReport.pairs_tested.offset,
                   pgo.PcmReport.clique_rounds.offset, pgo.PcmReport.clique_ms.offset] == [24, 16, 56, 8, 24, 48]
    from d2slam_b200.solver import lib
    cfg = pgo.PcmConfig()
    assert lib().d2pgo_default_pcm_config(C.byref(cfg)) == 0
    assert (cfg.pcm_thres, cfg.pos_covariance_per_meter, cfg.yaw_covariance_per_meter) == (1.635, 4e-3, 4e-5)


def test_pcm_null_handle_is_refused():
    from d2slam_b200.solver import lib
    assert lib().d2pgo_pcm(None, None, 0, None, None, None, 0, None, None, None, None, None, None) == 1


# ----------------------------------------------------------------------------------------------- GPU
def _run(s, case, is4=None, rel_key="rel_bad", **cfg):
    return s.pcm(case["frame_ids"], case["frame_agent"], case["ego"], case["kf_a"], case["kf_b"], case[rel_key], case["sqrt_info"], **cfg)


def _cfg(name):
    is4, thr, pc, yc = PCM_CONFIGS[name]
    return is4, dict(pcm_thres=thr, pos_covariance_per_meter=pc, yaw_covariance_per_meter=yc)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_device_pcm_matches_golden_reference(name):
    z = _gold(); case = _gold_case()
    is4, cfg = _cfg(name)
    s = pgo.PgoSolver(pose_dof=4 if is4 else 6)
    good = _run(s, case, **cfg)
    smd = s.debug_pcm_smd(); want = z[f"{name}_smd"]
    assert smd.shape == want.shape
    assert np.all(np.abs(smd - want) <= 1e-9 * np.abs(want))
    thr = float(np.float32(cfg["pcm_thres"]))
    assert not np.any(np.abs(want - thr) <= 1e-9 * thr)   # no bit is decided by rounding
    assert np.array_equal(good, z[f"{name}_good"])
    r = s.pcm_report
    n = len(case["kf_a"])
    assert r.inliers == good.sum() and r.pairs_tested == len(want) and r.consistent_pairs == int((want < thr).sum())


@pytest.mark.gpu
def test_device_clique_equals_golden_fmc():
    gs, cs = _gold_graphs()
    s = pgo.PgoSolver()
    for A, want in zip(gs, cs):
        assert np.nonzero(s.debug_pcm_clique(A))[0].tolist() == want


@pytest.mark.gpu
def test_device_pcm_is_bitwise_reproducible():
    g = pgo.make_pose_graph(seed=2, n_agents=4, poses_per_agent=300, loops=1500)
    c = pgo.make_pcm_case(g, 0.05, seed=3)
    s = pgo.PgoSolver(pose_dof=4)
    m1 = _run(s, c, pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2); d1 = s.debug_pcm_smd(); r1 = s.pcm_report.clique_rounds
    m2 = _run(s, c, pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2); d2 = s.debug_pcm_smd()
    assert np.array_equal(m1, m2) and d1.tobytes() == d2.tobytes() and r1 == s.pcm_report.clique_rounds


@pytest.mark.gpu
@pytest.mark.parametrize("is4", [0, 1])
def test_device_pcm_medium_case_matches_oracle(is4):
    g = pgo.make_pose_graph(seed=8, n_agents=3, poses_per_agent=500, loops=3000)
    c = pgo.make_pcm_case(g, 0.05, seed=9)
    s = pgo.PgoSolver(pose_dof=4 if is4 else 6)
    good = _run(s, c, pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2)
    want, smd = po.pcm(c, is4, 3.5, 0.5, 1e-2, rel_key="rel_bad")
    dev = s.debug_pcm_smd()
    assert np.all(np.abs(dev - smd) <= 1e-9 * np.abs(smd))
    thr = float(np.float32(3.5))
    assert not np.any(np.abs(smd - thr) <= 1e-9 * thr)
    assert np.array_equal(good, want)


@pytest.mark.gpu
def test_device_pcm_refuses_bad_input():
    case = small_case()
    s = pgo.PgoSolver()
    for kw in (dict(pcm_thres=float("nan")), dict(pcm_thres=0.0), dict(pcm_thres=-1.0), dict(pcm_thres=float("inf"))):
        with pytest.raises(RuntimeError, match="pcm_thres"):
            _run(s, case, **kw)
    bad = dict(case); bad["kf_a"] = np.array(case["kf_a"]); bad["kf_a"][3] = 999_999_999
    with pytest.raises(RuntimeError, match="unknown keyframe id 999999999"):
        _run(s, bad)
    n = 32769   # one group larger than the limit: every loop between frames 0 and 1 of drone 0
    big = dict(frame_ids=np.array([0, 1], np.int64), frame_agent=np.zeros(2, np.int32), ego=np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)),
               kf_a=np.zeros(n, np.int64), kf_b=np.ones(n, np.int64), rel_bad=np.tile([1.0, 0, 0, 0, 0, 0, 1], (n, 1)), sqrt_info=np.tile(np.eye(6).ravel(), (n, 1)))
    with pytest.raises(RuntimeError, match="32769 loops; at most 32768"):
        _run(s, big)


@pytest.mark.gpu
def test_4dof_pcm_then_solve_removes_the_outliers_damage():
    """PCM on the device, the inliers added to a 4-DoF handle, solved; against the oracle's PCM then solve_4d.  The same solve
    with every loop (outliers included) ends further from the ground truth."""
    g = pgo.make_pose_graph(seed=21, n_agents=3, poses_per_agent=80, loops=240)
    c = pgo.make_pcm_case(g, 0.05, seed=22)
    h = pgo.pose_graph_to_4d(g, seed=23)
    n_odo = c["n_odo"]
    bad_idx = n_odo + np.nonzero(c["outlier"])[0]
    h["rel"][bad_idx, :3] += c["bad_dt"]; h["rel"][bad_idx, 3] = pgo.normalize_angle(h["rel"][bad_idx, 3] + c["bad_yaw"])
    s = pgo.PgoSolver(pose_dof=4)
    good = _run(s, c, pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2)
    want, _ = po.pcm(c, 1, 3.5, 0.5, 1e-2, rel_key="rel_bad")
    assert np.array_equal(good, want) and not (good & c["outlier"]).any()
    keep = np.concatenate([np.ones(n_odo, bool), good])

    def solve(mask):
        t = pgo.PgoSolver(pose_dof=4, max_iterations=100, pcg_max_iterations=3000, pcg_tolerance=1e-13, lambda0=0.0, function_tolerance=1e-15)
        t.set_poses_4d(h["ids"], h["init"], h["fixed"])
        t.add_edges_4d(h["id_a"][mask], h["id_b"][mask], h["rel"][mask], h["sqrt_info"][mask])
        t.solve()
        return t.get_poses_4d(h["ids"])

    def err(x):
        return float(np.sqrt(np.mean(np.sum((x[:, :3] - h["gt"][:, :3]) ** 2, axis=1))))
    x = solve(keep)
    x_ref, _ = p4.solve_4d(h["init"], h["fixed"], h["ea"][keep], h["eb"][keep], h["rel"][keep], h["sqrt_info"][keep], iters=60)
    dp = np.abs(x[:, :3] - x_ref[:, :3]).max(); dyaw = np.abs(pgo.normalize_angle(x[:, 3] - x_ref[:, 3])).max()
    assert dp <= 1e-6 and dyaw <= 1e-6, (dp, dyaw)
    x_all = solve(np.ones(len(keep), bool))
    e_pcm, e_all = err(x), err(x_all)
    print(f"position RMSE to ground truth: with PCM {e_pcm:.4f} m, without {e_all:.4f} m")
    assert e_pcm < 0.5 * e_all, (e_pcm, e_all)
