"""PCM as a stream (include/d2pgo.h d2pgo_pcm_stream): the numpy restatement (oracle/pcm_stream_oracle.py PcmStream, fmc_heu_inc)
pinned to the reference's own SwarmLocalOutlierRejection kept across calls and FMC::maxCliqueHeuIncremental (live through
oracle/_ref where the reference tree exists, and through tests/golden/ref_pcm_stream.npz everywhere), and the device against
both and against d2pgo_pcm on the concatenated input."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pcm_oracle as po
from oracle import pcm_stream_oracle as pso
from oracle import ref_pcm_stream as ref
from test_pgo_pcm import PCM_CONFIGS, fmc_graphs, small_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_pcm_stream.npz")
LIVE = pytest.mark.skipif(not ref.available(), reason="reference PCM library not built")
WIDE = dict(pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2)


def batchings(case):
    """Named splits of a make_pcm_case input into calls, each a list of (frame indices, indices of the loops new in the call):
    one call; 7 and 23 arrival steps (pgo.pcm_arrival_steps); every frame first, then one loop per call."""
    n = len(case["kf_a"])
    one = [(np.arange(len(case["frame_ids"])), np.arange(n))]
    each = [(np.arange(len(case["frame_ids"])), np.zeros(0, np.int64))] + [(np.zeros(0, np.int64), np.array([e])) for e in range(n)]
    return {"one_call": one, "steps7": pgo.pcm_arrival_steps(case, 7), "steps23": pgo.pcm_arrival_steps(case, 23), "loop_each": each}


def cumulative(calls):
    """(frames, every loop so far) per call: the loops D2PGO passes on each call."""
    seen = np.zeros(0, np.int64)
    for f, l in calls:
        seen = np.concatenate([seen, np.asarray(l, np.int64)])
        yield np.asarray(f, np.int64), seen


def fmc_inc_graphs(seed=5):
    """fmc_graphs() with (num_new, prev) pairs: all new and prev 0, no new vertex, prev above, at and below the best."""
    rng = np.random.default_rng(seed)
    graphs, new, prev = [], [], []
    for A in fmc_graphs():
        n = len(A)
        for num_new, p in ((n, 0), (0, 0), (int(rng.integers(1, n + 1)), 0), (int(rng.integers(0, n + 1)), int(rng.integers(0, 6))),
                           (int(rng.integers(1, n + 1)), int(rng.integers(1, max(2, n // 2))))):
            graphs.append(A); new.append(num_new); prev.append(p)
    return graphs, new, prev


def _gold():
    return np.load(GOLD)


def _split(a, counts):
    return np.split(a, np.cumsum(counts)[:-1]) if len(counts) else []


def _oracle_run(case, calls, is4, thr, pc, yc, inc=0):
    s = pso.PcmStream(is4, thr, pc, yc, inc)
    return [s.call(*pgo.pcm_stream_args(case, f, l)) for f, l in cumulative(calls)]


def _ref_order(d):
    return np.concatenate([d[k] for k in sorted(d)]) if d else np.zeros(0)


# ----------------------------------------------------------------------------------------------- CPU
def test_golden_stream_inputs_are_the_test_batchings():
    z, case = _gold(), small_case()
    for b, calls in batchings(case).items():
        assert np.array_equal(z[f"{b}_frames"], np.concatenate([f for f, _ in calls])), b
        assert np.array_equal(z[f"{b}_loops"], np.concatenate([l for _, l in calls])), b
        assert np.array_equal(z[f"{b}_n_loops"], [len(l) for _, l in calls]), b
    g, k, p = fmc_inc_graphs()
    assert np.array_equal(z["inc_new"], k) and np.array_equal(z["inc_prev"], p)
    assert np.array_equal(z["inc_adj"], np.concatenate([a.ravel() for a in g]))


def test_arrival_steps_reveal_frames_in_order_and_loops_once_both_frames_exist():
    case = small_case()
    steps = pgo.pcm_arrival_steps(case, 23)
    frames = np.concatenate([f for f, _ in steps]); loops = np.concatenate([l for _, l in steps])
    assert sorted(frames.tolist()) == list(range(len(case["frame_ids"]))) and sorted(loops.tolist()) == list(range(len(case["kf_a"])))
    agent = np.asarray(case["frame_agent"])
    for a in np.unique(agent):
        assert np.all(np.diff(frames[agent[frames] == a]) > 0)   # each drone's trajectory in order
    fidx = {int(f): k for k, f in enumerate(case["frame_ids"])}
    shown = set()
    for f, l in steps:
        shown |= set(f.tolist())
        for e in l:
            assert fidx[int(case["kf_a"][e])] in shown and fidx[int(case["kf_b"][e])] in shown
    for t, (f, l) in enumerate(steps[1:]):   # no loop could have arrived a step earlier
        prev = set(np.concatenate([g for g, _ in steps[: t + 1]]).tolist())
        assert not any(fidx[int(case["kf_a"][e])] in prev and fidx[int(case["kf_b"][e])] in prev for e in l)


@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_oracle_stream_matches_golden_reference(name):
    z, case = _gold(), small_case()
    is4, thr, pc, yc = PCM_CONFIGS[name]
    for b, calls in batchings(case).items():
        got = _oracle_run(case, calls, is4, thr, pc, yc)
        n_call = [len(l) for _, l in cumulative(calls)]
        for (m, d), want_m, want_s in zip(got, _split(z[f"{b}_{name}_good"], n_call), _split(z[f"{b}_{name}_smd"], z[f"{b}_{name}_n_smd"])):
            assert np.array_equal(m, want_m), b
            s = _ref_order(d)
            assert s.shape == want_s.shape and np.all(np.abs(s - want_s) <= 1e-10 * np.abs(want_s)), b


@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_oracle_stream_mode0_equals_the_batch_oracle(name):
    case = small_case()
    is4, thr, pc, yc = PCM_CONFIGS[name]
    for b, calls in batchings(case).items():
        order = np.concatenate([l for _, l in calls])
        cc = dict(case, kf_a=case["kf_a"][order], kf_b=case["kf_b"][order], rel_bad=case["rel_bad"][order], sqrt_info=case["sqrt_info"][order])
        want, _ = po.pcm(cc, is4, thr, pc, yc, rel_key="rel_bad")
        assert np.array_equal(_oracle_run(case, calls, is4, thr, pc, yc)[-1][0], want), b


@LIVE
def test_reference_pin_reproduces_its_golden_file():
    """The live libd2ref_pcm_stream.so recomputes tests/golden/ref_pcm_stream.npz bit for bit (as tests/test_ref_frozen.py
    does for the other pins): same keys, dtype, shape and bytes."""
    import importlib
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    live = {k: np.asarray(v) for k, v in importlib.import_module("make_ref_pcm_stream_golden").arrays().items()}
    with np.load(GOLD) as g:
        frozen = {k: g[k] for k in g.files}
    assert sorted(live) == sorted(frozen)
    assert [k for k in live if not (live[k].dtype == frozen[k].dtype and live[k].shape == frozen[k].shape and live[k].tobytes() == frozen[k].tobytes())] == []


@LIVE
@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_oracle_stream_matches_live_reference(name):
    case = small_case()
    is4, thr, pc, yc = PCM_CONFIGS[name]
    for b, calls in batchings(case).items():
        o = pso.PcmStream(is4, thr, pc, yc); r = ref.PcmStream(is4, thr, pc, yc)
        for f, l in cumulative(calls):
            args = pgo.pcm_stream_args(case, f, l)
            (m, d), (mr, sr) = o.call(*args), r.call(*args)
            assert np.array_equal(m, mr), b
            s = _ref_order(d)
            assert s.shape == sr.shape and np.all(np.abs(s - sr) <= 1e-10 * np.abs(sr)), b


def _is_clique(A, c):
    c = list(c)
    return all(A[u, v] for i, u in enumerate(c) for v in c[i + 1:])


def test_oracle_incremental_clique_matches_golden_fmc():
    z = _gold()
    g, k, p = fmc_inc_graphs()
    beaten = 0
    for A, num_new, prev, want in zip(g, k, p, z["inc_ret"]):
        size, best = pso.fmc_heu_inc(A, num_new, prev)
        assert size == want
        n = len(A)
        if best:
            beaten += 1
            assert len(best) == size > prev and _is_clique(A, best) and len(set(best)) == len(best)
            assert any(v >= n - num_new for v in best)
        else:
            assert size == prev
        if num_new == n and prev == 0:
            assert best == po.fmc_heu(A)
    assert 0 < beaten < len(g)


@LIVE
def test_oracle_incremental_clique_matches_live_fmc():
    for A, num_new, prev in zip(*fmc_inc_graphs(seed=9)):
        assert pso.fmc_heu_inc(A, num_new, prev)[0] == ref.fmc_heu_inc(A, num_new, prev)


def test_oracle_stream_mode1_sets_never_shrink_and_reject_every_outlier():
    case = small_case()
    for name in ("d6_wide", "d4_wide"):
        is4, thr, pc, yc = PCM_CONFIGS[name]
        for b, calls in batchings(case).items():
            s = pso.PcmStream(is4, thr, pc, yc, 1); sizes = {}
            for f, l in cumulative(calls):
                m, _ = s.call(*pgo.pcm_stream_args(case, f, l))
                for key, mem in s.members.items():
                    assert len(mem) >= sizes.get(key, 0)
                    sizes[key] = len(mem)
            assert not (m & case["outlier"][l]).any(), (name, b)


def test_pcm_stream_report_layout():
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "d2pgo.h"\nint main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(d2pgo_pcm_stream_report), '
            'offsetof(d2pgo_pcm_stream_report, inliers), offsetof(d2pgo_pcm_stream_report, pairs_tested), offsetof(d2pgo_pcm_stream_report, device_ms), '
            'offsetof(d2pgo_pcm_stream_report, clique_ms));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "t.c"); exe = os.path.join(td, "t")
        open(c, "w").write(code)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = list(map(int, subprocess.check_output([exe]).decode().split()))
    R = pgo.PcmStreamReport
    assert out == [C.sizeof(R), R.inliers.offset, R.pairs_tested.offset, R.device_ms.offset, R.clique_ms.offset] == [72, 16, 24, 48, 64]


def test_pcm_stream_null_handle_is_refused():
    from d2slam_b200.solver import lib
    L = lib()
    assert L.d2pgo_pcm_stream_reset(None, None, 0) == 1
    assert L.d2pgo_pcm_stream(None, 0, None, None, None, 0, None, None, None, None, None, None, None) == 1
    assert L.d2pgo_debug_pcm_stream_smd(None, None, 0) == 1
    assert L.d2pgo_debug_pcm_clique_inc(None, 0, None, 0, 0, None, None) == 1


# ----------------------------------------------------------------------------------------------- GPU
def _cfg(name):
    is4, thr, pc, yc = PCM_CONFIGS[name]
    return is4, dict(pcm_thres=thr, pos_covariance_per_meter=pc, yaw_covariance_per_meter=yc)


def _stream(s, case, calls, rel_key="rel_bad"):
    """Runs calls on s (already reset) -> per call (mask over every loop so far, smd of the call, report)."""
    out = []
    for f, l in cumulative(calls):
        m = s.pcm_stream(*pgo.pcm_stream_args(case, f, l, rel_key))
        out.append((m, s.debug_pcm_stream_smd(), s.pcm_stream_report))
    return out


def _group_major(case, calls, smds):
    """The smd the stream gathered over the calls, in d2pgo_pcm's order on the concatenated input: per group (in order of
    its first loop) every row's pairs, rows ascending."""
    agent = np.asarray(case["frame_agent"]); fidx = {int(f): k for k, f in enumerate(case["frame_ids"])}
    gid, size, parts = {}, [], []
    for (_, l), smd in zip(calls, smds):
        new = {}
        for e in l:
            x, y = agent[fidx[int(case["kf_a"][e])]], agent[fidx[int(case["kf_b"][e])]]
            g = gid.setdefault((min(x, y), max(x, y)), len(gid))
            if g == len(size):
                size.append(0); parts.append([])
            new[g] = new.get(g, 0) + 1
        o = 0
        for g in sorted(new):
            L0 = size[g]; L = L0 + new[g]; k = L * (L - 1) // 2 - L0 * (L0 - 1) // 2
            parts[g].append(smd[o:o + k]); o += k; size[g] = L
        assert o == len(smd)
    return np.concatenate([np.concatenate(p) for p in parts]) if parts else np.zeros(0)


def _concat_batch(s, case, calls, cfg):
    order = np.concatenate([l for _, l in calls])
    m = s.pcm(case["frame_ids"], case["frame_agent"], case["ego"], case["kf_a"][order], case["kf_b"][order], case["rel_bad"][order],
              case["sqrt_info"][order], **cfg)
    return m, s.debug_pcm_smd()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PCM_CONFIGS))
def test_device_stream_mode0_matches_golden_reference(name):
    z, case = _gold(), small_case()
    is4, cfg = _cfg(name)
    s = pgo.PgoSolver(pose_dof=4 if is4 else 6)
    for b, calls in batchings(case).items():
        s.pcm_stream_reset(0, **cfg)
        got = _stream(s, case, calls)
        orc = _oracle_run(case, calls, *PCM_CONFIGS[name])   # which groups each call touched, for the reference's group order
        n_call = [len(l) for _, l in cumulative(calls)]
        order = _first_loop_order(case, calls)
        for (m, smd, r), (_, d), want_m, want_s in zip(got, orc, _split(z[f"{b}_{name}_good"], n_call), _split(z[f"{b}_{name}_smd"], z[f"{b}_{name}_n_smd"])):
            assert np.array_equal(m, want_m), b
            first = [k for k in order if k in d]   # the device lists a call's groups in order of their first loop
            sizes = {k: len(d[k]) for k in d}
            off = np.cumsum([0] + [sizes[k] for k in first]); dev = {k: smd[off[i]:off[i + 1]] for i, k in enumerate(first)}
            got_ref = _ref_order(dev)
            assert got_ref.shape == want_s.shape and np.all(np.abs(got_ref - want_s) <= 1e-9 * np.abs(want_s)), b
            assert r.pairs_tested == len(want_s) and r.inliers == m.sum()


def _first_loop_order(case, calls):
    """Group keys (max drone, min drone) in order of their first loop over the calls."""
    agent = np.asarray(case["frame_agent"]); fidx = {int(f): k for k, f in enumerate(case["frame_ids"])}
    keys = {}
    for _, l in calls:
        for e in l:
            x, y = agent[fidx[int(case["kf_a"][e])]], agent[fidx[int(case["kf_b"][e])]]
            keys.setdefault((max(x, y), min(x, y)), None)
    return list(keys)


def _one_group_case(n_loops=1100):
    """One drone, so every loop falls into one group: enough loops to carry it across the pitch growth at 32 and 1024."""
    g = pgo.make_pose_graph(seed=31, n_agents=1, poses_per_agent=400, loops=n_loops)
    return pgo.make_pcm_case(g, 0.05, seed=32)


def _pitch_batches(case):
    n = len(case["kf_a"]); f = np.arange(len(case["frame_ids"]))
    cuts = [0, 31, 33, 600, 1023, 1025, n]
    return [(f if k == 0 else np.zeros(0, np.int64), np.arange(a, b)) for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))]


@pytest.mark.gpu
@pytest.mark.parametrize("is4", [0, 1])
def test_device_stream_mode0_is_bitwise_the_batch_on_the_concatenated_input(is4):
    """After any split into calls, the last mask and the smd gathered over the calls are bitwise d2pgo_pcm's on the
    concatenated input: one call, one loop per call, arrival steps, and calls that carry a group across the pitch growth."""
    small, big = small_case(), _one_group_case()
    g = pgo.make_pose_graph(seed=8, n_agents=3, poses_per_agent=300, loops=1500)
    med = pgo.make_pcm_case(g, 0.05, seed=9)
    assert len(big["kf_a"]) > 1025
    runs = [(small, c) for c in batchings(small).values()] + [(med, pgo.pcm_arrival_steps(med, 100)), (big, _pitch_batches(big))]
    s = pgo.PgoSolver(pose_dof=4 if is4 else 6)
    for case, calls in runs:
        s.pcm_stream_reset(0, **WIDE)
        got = _stream(s, case, calls)
        want_m, want_s = _concat_batch(s, case, calls, WIDE)
        assert np.array_equal(got[-1][0], want_m)
        assert _group_major(case, calls, [x[1] for x in got]).tobytes() == want_s.tobytes()
        assert sum(r.pairs_tested for _, _, r in got) == len(want_s) and got[-1][2].total_loops == len(want_m)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d6_wide", "d4_wide", "d6_default"])
def test_device_stream_mode1_sets_are_the_oracles(name):
    case = small_case()
    is4, cfg = _cfg(name)
    s = pgo.PgoSolver(pose_dof=4 if is4 else 6)
    g = pgo.make_pose_graph(seed=8, n_agents=3, poses_per_agent=300, loops=1500)
    med = pgo.make_pcm_case(g, 0.05, seed=9)
    runs = [(case, c) for c in batchings(case).values()] + [(med, pgo.pcm_arrival_steps(med, 40))]
    for c, calls in runs:
        s.pcm_stream_reset(1, **cfg)
        o = pso.PcmStream(*PCM_CONFIGS[name], incremental=1)
        sizes = {}
        for (f, l), (m, _, r) in zip(cumulative(calls), _stream(s, c, calls)):
            want, _ = o.call(*pgo.pcm_stream_args(c, f, l))
            assert np.array_equal(m, want)   # every group's set, loop by loop
            for key, mem in o.members.items():
                assert len(mem) >= sizes.get(key, 0)
                sizes[key] = len(mem)
            assert r.inliers == want.sum()
        if c is case:
            assert not (m & c["outlier"][l]).any()


@pytest.mark.gpu
def test_device_incremental_clique_matches_golden_fmc():
    z = _gold()
    s = pgo.PgoSolver()
    for A, num_new, prev, want in zip(*fmc_inc_graphs(), z["inc_ret"]):
        member, size = s.debug_pcm_clique_inc(A, num_new, prev)
        assert size == want
        assert np.nonzero(member)[0].tolist() == sorted(pso.fmc_heu_inc(A, num_new, prev)[1])


@pytest.mark.gpu
def test_device_streams_are_bitwise_reproducible():
    g = pgo.make_pose_graph(seed=2, n_agents=4, poses_per_agent=300, loops=1500)
    c = pgo.make_pcm_case(g, 0.05, seed=3)
    calls = pgo.pcm_arrival_steps(c, 30)
    for inc in (0, 1):
        outs = []
        for _ in range(2):
            s = pgo.PgoSolver(pose_dof=4)
            s.pcm_stream_reset(inc, **WIDE)
            outs.append([(m.tobytes(), d.tobytes(), r.clique_rounds, r.consistent_pairs) for m, d, r in _stream(s, c, calls)])
        assert outs[0] == outs[1]


@pytest.mark.gpu
def test_device_stream_refusals_leave_the_stream_unchanged():
    case = small_case()
    calls = pgo.pcm_arrival_steps(case, 7)
    s0 = pgo.PgoSolver()
    with pytest.raises(RuntimeError, match="no d2pgo_pcm_stream_reset"):
        s0.pcm_stream(*pgo.pcm_stream_args(case, calls[0][0], calls[0][1]))
    for inc in (0, 1):
        want = pgo.PgoSolver(); want.pcm_stream_reset(inc, **WIDE); want_out = _stream(want, case, calls)
        s = pgo.PgoSolver(); s.pcm_stream_reset(inc, **WIDE)
        got = []
        for t, (f, l) in enumerate(cumulative(calls)):
            args = list(pgo.pcm_stream_args(case, f, l))
            if t == 3:
                fid, fag, ego, lid, ka, kb, rel, si = args
                bad = [("unknown keyframe id 999999", dict(ka=np.concatenate([ka, [999999]]), kb=np.concatenate([kb, kb[:1]]),
                                                          lid=np.concatenate([lid, [10 ** 6]]), rel=np.concatenate([rel, rel[:1]]), si=np.concatenate([si, si[:1]]))),
                       ("appears twice", dict(lid=np.concatenate([lid, lid[-1:]]), ka=np.concatenate([ka, ka[-1:]]), kb=np.concatenate([kb, kb[-1:]]),
                                              rel=np.concatenate([rel, rel[-1:]]), si=np.concatenate([si, si[-1:]]))),
                       ("now with drone", dict(fid=np.concatenate([fid, case["frame_ids"][:1]]), fag=np.concatenate([fag, [7]]), ego=np.concatenate([ego, ego[:1]]))),
                       ("non-finite relative pose", dict(rel=np.where(np.arange(len(rel))[:, None] == len(rel) - 1, np.nan, rel))),
                       ("non-finite ego pose", dict(ego=np.where(np.arange(len(ego))[:, None] == 0, np.inf, ego))),
                       ("non-finite sqrt_info", dict(si=np.where(np.arange(len(si))[:, None] == len(si) - 1, np.nan, si)))]
                for msg, kw in bad:
                    a = dict(fid=fid, fag=fag, ego=ego, lid=lid, ka=ka, kb=kb, rel=rel, si=si); a.update(kw)
                    with pytest.raises(RuntimeError, match=msg):
                        s.pcm_stream(a["fid"], a["fag"], a["ego"], a["lid"], a["ka"], a["kb"], a["rel"], a["si"])
                n = 32769   # a new group past the limit: loops between two frames of drone 0 already in the stream
                fr = np.asarray(case["frame_ids"])[calls[0][0][:2]]   # revealed by the first call
                with pytest.raises(RuntimeError, match="32769 loops; at most 32768"):
                    s.pcm_stream(np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros((0, 7)), 10 ** 7 + np.arange(n), np.full(n, fr[0]), np.full(n, fr[1]),
                                 np.tile([1.0, 0, 0, 0, 0, 0, 1], (n, 1)), np.tile(np.eye(6).ravel(), (n, 1)))
            m = s.pcm_stream(*args)
            got.append((m, s.debug_pcm_stream_smd(), s.pcm_stream_report))
        for (m, d, r), (wm, wd, wr) in zip(got, want_out):
            assert m.tobytes() == wm.tobytes() and d.tobytes() == wd.tobytes() and (r.pairs_tested, r.clique_rounds) == (wr.pairs_tested, wr.clique_rounds)


@pytest.mark.gpu
def test_device_stream_and_batch_interleave_on_one_handle():
    case = small_case()
    calls = pgo.pcm_arrival_steps(case, 7)
    a = pgo.PgoSolver(); a.pcm_stream_reset(0, **WIDE); want = _stream(a, case, calls)
    b = pgo.PgoSolver(); want_m = _run_batch(b, case); want_d = b.debug_pcm_smd()
    s = pgo.PgoSolver(); s.pcm_stream_reset(0, **WIDE)
    for (f, l), (wm, wd, _) in zip(cumulative(calls), want):
        m = s.pcm_stream(*pgo.pcm_stream_args(case, f, l))
        bm = _run_batch(s, case); bd = s.debug_pcm_smd()
        assert m.tobytes() == wm.tobytes() and s.debug_pcm_stream_smd().tobytes() == wd.tobytes()
        assert bm.tobytes() == want_m.tobytes() and bd.tobytes() == want_d.tobytes()


def _run_batch(s, case):
    return s.pcm(case["frame_ids"], case["frame_agent"], case["ego"], case["kf_a"], case["kf_b"], case["rel_bad"], case["sqrt_info"], **WIDE)
