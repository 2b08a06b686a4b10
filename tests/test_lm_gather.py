"""The landmark gather of single-drone windows with 96-byte records (k_lm_gather12, one lane per record) against the
128-byte-record path it replaces (k_lm_gather16, forced everywhere with D2BA_REC128=1), on batches that mix windows of
both formats, and the solves of such batches against the CPU oracle."""
import numpy as np
import pytest

from d2slam_b200 import abi, synth
from helpers import state_diff, state_of

pytestmark = pytest.mark.gpu

VIEWS = (abi.DBG_W, abi.DBG_HLL, abi.DBG_GL)


def bench_windows():
    """The windows of the bench workload (bench.make_batch: 11 frames, 300 landmarks, seeds from 1000)."""
    return [synth.make_window(seed=1000 + i) for i in range(3)]


def mixed_windows():
    """Eligible for 96-byte records: two bench windows and a far-off start whose fixed 8-iteration solve rejects a step.
    Not eligible: a window with constant poses (one-pose factors), a stereo window (1F2C factors), and a 40-frame window
    with landmarks of more than 32 records."""
    reject = synth.make_window(seed=81, n_landmarks=100, pose_noise=(1.0, np.deg2rad(15.0)))
    const = synth.make_window(seed=63, n_landmarks=80)
    pc = np.asarray(const["pose_const"], np.uint8).copy()
    pc[[0, 3]] = 1
    const["pose_const"] = pc
    stereo = synth.make_window(seed=64, cams="stereo", n_landmarks=80)
    long = synth.make_window(seed=65, n_frames=40, n_landmarks=60)
    assert np.unique(long["obs"]["landmark_id"], return_counts=True)[1].max() > 32
    b = bench_windows()
    return [b[0], reject, const, stereo, long, b[1]]


def make_solver(windows, monkeypatch, rec128, **cfg):
    from d2slam_b200.solver import Solver
    if rec128:
        monkeypatch.setenv("D2BA_REC128", "1")   # read by d2ba_create
    else:
        monkeypatch.delenv("D2BA_REC128", raising=False)
    s = Solver(max_windows=len(windows), **cfg)
    for i, p in enumerate(windows):
        p.load(s, i)
    s.finalize()
    return s


GATHERS = ("k_lm_gather12", "k_lm_gather16")


def gather_views(windows, monkeypatch, rec128):
    """DBG_W / DBG_HLL / DBG_GL of every window after one debug linearisation, each window's plan (D2BA_DBG_PLAN), and
    the gather kernels the linearisation launched.  A kernel counts when its (possibly mangled) name contains the kernel's
    name.  The device work is bracketed by synchronisations and 50 ms of host time inside the profiled region, so that
    no kernel record falls outside the profiler's window when the GPU and host clocks are a little apart: the
    linearisation of three bench windows lasts about a millisecond."""
    import time

    import torch
    from torch.profiler import ProfilerActivity, profile
    s = make_solver(windows, monkeypatch, rec128)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.05)
        s.debug_linearize()
        torch.cuda.synchronize()
        time.sleep(0.05)
    names = [e.name for e in prof.events()]
    out = [{item: s.debug_get(i, item) for item in VIEWS} for i in range(len(windows))]
    plans = [s.debug_plan(i) for i in range(len(windows))]
    s.close()
    return out, plans, {k for k in GATHERS if any(k in n for n in names)}


@pytest.mark.parametrize("batch", ["bench", "mixed"])
def test_rows_bitwise_equal_to_128_byte_records(batch, monkeypatch):
    windows = bench_windows() if batch == "bench" else mixed_windows()
    new, p_new, k_new = gather_views(windows, monkeypatch, rec128=False)
    old, p_old, k_old = gather_views(windows, monkeypatch, rec128=True)
    # the plan: 96-byte records and k_lm_gather12 chunks exactly where D2BA_REC128 is off and the window is eligible
    eligible = [i for i, p in enumerate(p_new) if p["rec_stride"] == 12]
    assert eligible == ([0, 1, 2] if batch == "bench" else [0, 1, 5]), [p["rec_stride"] for p in p_new]
    for i in range(len(windows)):
        assert (p_new[i]["n_g12"] > 0) == (i in eligible), (i, p_new[i])
        assert p_old[i]["n_g12"] == 0 and p_old[i]["rec_stride"] == (16 if i in eligible else p_new[i]["rec_stride"]), (i, p_old[i])
    # the kernels the linearisation launched
    assert "k_lm_gather12" in k_new and "k_lm_gather12" not in k_old, (k_new, k_old)
    assert "k_lm_gather16" in k_old
    if batch == "mixed":
        assert "k_lm_gather16" in k_new   # the ineligible windows keep their records and kernel
    for i in range(len(windows)):
        for item in VIEWS:
            a, b = new[i][item], old[i][item]
            assert a.shape == b.shape and np.isfinite(a).all(), (i, item)
            assert np.array_equal(a.view(np.int64), b.view(np.int64)), (i, item, float(np.abs(a - b).max()))


@pytest.mark.parametrize("rec128", [False, True])
def test_mixed_batch_solve_matches_oracle(rec128, monkeypatch):
    from oracle import orc
    windows = mixed_windows()
    iters = 8
    s = make_solver(windows, monkeypatch, rec128, max_num_iterations=iters)
    rs = s.solve_fixed(iters)
    rejected = 0
    for i, p in enumerate(windows):
        o = orc.Oracle(max_num_iterations=iters)
        p.load(o)
        ro = o.solve_fixed(iters)
        rejected += ro.total_iterations - ro.successful_steps
        assert ro.total_iterations == rs[i].total_iterations == iters
        assert ro.successful_steps == rs[i].successful_steps, i
        assert abs(rs[i].final_cost - ro.final_cost) <= 1e-7 * max(1.0, abs(ro.final_cost)), (i, rs[i].final_cost, ro.final_cost)
        d = state_diff(state_of(s, p, i), state_of(o, p))
        assert d["pos"] <= 1e-6 and d["rot"] <= 1e-6, (i, d)
        assert d["sb"] <= 1e-6 and d["lm_rel"] <= 1e-5 and d["ext_pos"] <= 1e-6 and d["td"] <= 1e-8, (i, d)
    assert rejected > 0


def test_admm_swarm_keeps_128_byte_records(monkeypatch):
    """The agents of an ADMM swarm (remote frames are leaves) are not eligible: the default path and D2BA_REC128=1 run
    the same kernels, and the solve matches the oracle's fixed-schedule ADMM."""
    from oracle import orc
    sw = synth.make_swarm(seed=83, n_agents=4, n_landmarks=120, shared_per_pair=20)
    steps, iters = 2, 4
    cfg = dict(consensus_max_steps=steps, max_num_iterations=iters)
    ags = []
    for p in sw:
        a = orc.Oracle(**cfg)
        p.load(a)
        ags.append(a)
    ro = orc.admm_solve(ags, fixed_mode=True)
    from torch.profiler import ProfilerActivity, profile
    s = make_solver(sw, monkeypatch, rec128=False, **cfg)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rs = s.solve_fixed(iters)
    assert not any("k_lm_gather12" in e.name for e in prof.events())
    for i, p in enumerate(sw):
        assert rs[i].total_iterations == ro[i].total_iterations
        assert abs(rs[i].final_cost - ro[i].final_cost) <= 1e-6 * max(1.0, ro[i].final_cost), (i, rs[i].final_cost, ro[i].final_cost)
        d = state_diff(state_of(s, p, i), state_of(ags[i], p))
        assert d["pos"] <= 1e-6 and d["rot"] <= 1e-6 and d["lm_rel"] <= 1e-5, (i, d)
