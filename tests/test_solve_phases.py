"""Phase timestamps of the one-kernel reduced-system solve (k_solve_small's timestamped instantiation, read through
d2ba_debug_solve_phases): what tools/solve_tail_probe.py splits the kernel's time by."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def bench_solver(iters):
    """A handle of 4 bench windows (11 frames, 300 landmarks) per SM: one wave of k_solve_small."""
    import torch
    from d2slam_b200 import synth
    from d2slam_b200.solver import Solver
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count
    s = Solver(max_windows=n, max_num_iterations=iters)
    for i in range(n):
        synth.make_window(seed=1000 + i, n_frames=11, n_landmarks=300).load(s, i)
    s.finalize()
    return s


def test_phase_timestamps(monkeypatch):
    """Each window's five timestamps are in order, and the span they cover is the kernel's: the windows run in one wave,
    so no window runs outside the launch's event time and the median window's span is within 10 % of it."""
    monkeypatch.delenv("D2BA_NO_FUSED_SOLVE", raising=False)
    s = bench_solver(4)
    assert s.solve_occupancy() == 4
    ts, ms = s.solve_phases(4)
    n = s.num_windows()
    s.close()
    assert ts.shape == (4, n, 5)
    full = 0
    for it in range(4):
        t = ts[it]
        ran = t[:, 0] > 0
        assert ran.sum() > n // 2, it
        assert (np.diff(t[ran], axis=1) >= 0).all(), it
        full += int((t[ran, 2] > t[ran, 1]).sum())   # windows that ran the Cholesky (not a rejected-step reuse)
        launch_ns = ms[it] * 1e6
        span = t[ran, 4].max() - t[ran, 0].min()
        median = np.median(t[ran, 4] - t[ran, 0])
        assert span <= launch_ns * 1.01, (it, span, launch_ns)
        assert median >= 0.9 * launch_ns, (it, median, launch_ns)
    assert full > 0


def test_phase_timestamps_need_finalize():
    from d2slam_b200.solver import D2BAError, Solver
    s = Solver(max_windows=1)
    with pytest.raises(D2BAError):
        s.solve_phases(1)
    s.close()
