"""Where the back half of a trust-region iteration of the bench workload spends its time: the reduced-system solve
(Schur complement, Cholesky, speed-bias back-substitution) and the step, either as the one kernel k_solve_small or as
the separate kernels k_schur_small -> k_chol_smem -> k_sb_back -> k_step (D2BA_NO_FUSED_SOLVE=1).

Runs the flagship workload of bench.py (make_batch(528, 1000), 8 fixed iterations, device-resident solve_fixed) once per
path, each in its own handle, takes one torch.profiler trace (CUDA activities) of a CUDA-graph replay and reports:
  - device time per launch of each tail kernel;
  - the tail span per iteration, from the start of the Schur kernel (or k_solve_small) to the end of the step kernel;
  - the bytes the tail has to move per iteration, computed from the shapes (the Schur pass reads the landmark rows Wt
    and the eliminated speed-bias rows Y, the speed-bias back-substitution reads Y again and its L / E blocks, the step
    reads the landmark rows again: the same for both paths), and the resulting GB/s over the tail span;
  - the CTAs per SM of k_solve_small (cudaOccupancyMaxActiveBlocksPerMultiprocessor at the handle's shared memory);
  - "phases" (fused path): k_solve_small's four phases from its timestamped instantiation (d2ba_debug_solve_phases),
    per-window durations, the spread of the Cholesky start across windows, and the batch GB/s of each streaming phase.

    python tools/solve_tail_probe.py --out DIR [--batch 528] [--iters 8] [--paths separate,fused]

Traces go to DIR/tail_{fused,separate}.pt.trace.json and the summary to DIR/solve_tail.json (also printed).  The tree
the script sits in is the one imported, so a copy of the script inside another checkout measures that checkout (a
checkout without the fused kernel reports its separate kernels twice).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAIL = ("k_schur_small", "k_chol_smem", "k_sb_back", "k_step", "k_solve_small")


def short(n):
    n = n.split("(")[0].split("<")[0]
    return n.replace("void ", "").replace("d2ba::", "").strip()


def phase_bytes(s, probs):
    """Bytes each streaming phase of the tail reads per window, from the shapes: [(Schur, sb back, step)] per window."""
    import numpy as np
    from d2slam_b200 import abi
    out = []
    for i, p in enumerate(probs):
        nlc = int(np.asarray(s.debug_get(i, abi.DBG_N_LC, np.int64)).reshape(-1)[0])
        n_c = int(np.asarray(s.debug_get(i, abi.DBG_N_CAM, np.int64)).reshape(-1)[0])
        nl, nb = len(p["lm_ids"]), (n_c - nlc) // 9
        ldw = (nlc + 1 + 7) // 8 * 8
        wt_rows = (nl + 9 * nb + 31) // 32 * 32
        out.append((wt_rows * ldw * 8, (9 * nb * (nlc + 1) + 171 * nb) * 8, nl * ldw * 8))
    return out


def tail_bytes(s, probs):
    return sum(sum(b) for b in phase_bytes(s, probs))


def pct(v, q):
    import numpy as np
    return round(float(np.percentile(v, q)), 2)


def phases(s, probs, args):
    """k_solve_small per phase, from its timestamped instantiation (d2ba_debug_solve_phases) over args.iters fixed
    iterations: duration of each phase per window (median, 10th / 90th percentile, min / max over the windows that ran
    all four), the spread of the phase-2 start times across windows per launch, and the batch rate of each streaming
    phase (its bytes over the span from the first window's start to the last window's end of that phase)."""
    import numpy as np
    import bench
    bench.reset_state(s, probs)
    ts, ms = s.solve_phases(args.iters)
    pb = np.array(phase_bytes(s, probs), dtype=np.float64)   # [window, (1, 3, 4)]
    names = ("schur", "chol", "sb_back", "step")
    dur = {n: [] for n in names}
    start2, rate, span_sum = [], {n: [] for n in ("schur", "sb_back", "step")}, []
    for it in range(ts.shape[0]):
        t = ts[it].astype(np.float64)
        full = (t[:, 0] > 0) & (t[:, 1] > t[:, 0]) & (t[:, 2] > t[:, 1])   # ran phases (1)-(3): not a rejected-step reuse
        if not full.any():
            continue
        tf = t[full]
        for k, n in enumerate(names):
            dur[n].extend(((tf[:, k + 1] - tf[:, k]) * 1e-3).tolist())
        start2.append((tf[:, 1].max() - tf[:, 1].min()) * 1e-3)
        for k, n, j in ((0, "schur", 0), (2, "sb_back", 1), (3, "step", 2)):
            span = (tf[:, k + 1].max() - tf[:, k].min()) * 1e-9
            rate[n].append(pb[full, j].sum() / span / 1e9)
        ran = t[:, 0] > 0
        span_sum.append({"launch_us": round(ms[it] * 1e3, 2), "windows_span_us": round((t[ran, 4].max() - t[ran, 0].min()) * 1e-3, 2),
                         "median_window_us": round(float(np.median(t[ran, 4] - t[ran, 0])) * 1e-3, 2)})
    res = {"iterations_with_full_solves": len(start2)}
    for n in names:
        v = dur[n]
        res[n + "_us"] = {"median": pct(v, 50), "p10": pct(v, 10), "p90": pct(v, 90), "min": pct(v, 0), "max": pct(v, 100)} if v else None
    res["chol_start_spread_us"] = {"median": pct(start2, 50), "min": pct(start2, 0), "max": pct(start2, 100)} if start2 else None
    res["bytes_per_window"] = {"schur": int(pb[:, 0].mean()), "sb_back": int(pb[:, 1].mean()), "step": int(pb[:, 2].mean())}
    res["batch_gbs"] = {n: pct(v, 50) if v else None for n, v in rate.items()}
    res["launches"] = span_sum
    return res


def run(path, args, probs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from d2slam_b200.solver import Solver
    if path == "separate":
        os.environ["D2BA_NO_FUSED_SOLVE"] = "1"   # read by d2ba_create
    else:
        os.environ.pop("D2BA_NO_FUSED_SOLVE", None)
    s = Solver(max_windows=args.batch, max_num_iterations=args.iters)
    bench.load_all(s, probs)
    s.finalize()
    occ = s.solve_occupancy() if hasattr(s, "solve_occupancy") else None
    for _ in range(3):   # the iteration graph is captured from the second solve on
        bench.reset_state(s, probs)
        s.solve_fixed(args.iters)
    torch.cuda.synchronize()
    bench.reset_state(s, probs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.solve_fixed(args.iters)
        torch.cuda.synchronize()
    trace = os.path.join(args.out, f"tail_{path}.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])
    k = [(short(e["name"]), float(e["ts"]), float(e["ts"]) + float(e["dur"])) for e in ev]
    per = {}
    for n, a, b in k:
        if n in TAIL:
            d = per.setdefault(n, [0, 0.0])
            d[0] += 1
            d[1] += b - a
    spans, t0 = [], None
    for n, a, b in k:
        if n in ("k_schur_small", "k_solve_small") and t0 is None:
            t0 = a
        if n in ("k_step", "k_solve_small") and t0 is not None:
            spans.append(b - t0)
            t0 = None
    nbytes = tail_bytes(s, probs)
    ph = phases(s, probs, args) if path == "fused" and occ else None
    s.close()
    span = sum(spans) / len(spans) if spans else None
    return {
        "kernel_us_per_launch": {n: round(v[1] / v[0], 2) for n, v in per.items()},
        "launches": {n: v[0] for n, v in per.items()},
        "tails": len(spans),
        "tail_span_us_per_iteration": round(span, 2) if span else None,
        "tail_bytes_per_iteration": nbytes,
        "tail_gbs": round(nbytes / (span * 1e-6) / 1e9, 1) if span else None,
        "k_solve_small_ctas_per_sm": occ,
        "phases": ph,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=528)
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--paths", default="separate,fused", help="comma-separated subset of separate,fused")
    args = ap.parse_args()
    import torch
    import bench

    if not torch.cuda.is_available():
        sys.exit("solve_tail_probe: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    probs = bench.make_batch(args.batch, 1000)
    res = {"gpu": torch.cuda.get_device_name(0), "batch": args.batch, "iters": args.iters}
    for path in args.paths.split(","):
        res[path] = run(path, args, probs)
    if "separate" in res and "fused" in res:
        a, b = res["separate"]["tail_span_us_per_iteration"], res["fused"]["tail_span_us_per_iteration"]
        res["fused_over_separate_span"] = round(b / a, 3) if a and b else None
    with open(os.path.join(args.out, "solve_tail.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
