"""Where the landmark hand-off of the bench workload spends its time.

Runs the flagship workload of bench.py (make_batch(528, 1000), 8 fixed iterations, device-resident solve_fixed), takes
one torch.profiler trace (CUDA activities) of a CUDA-graph replay and reports, per launch (one gather / Schur
elimination per trust-region iteration, one more reprojection pass for the initial linearisation):
  - device time of the landmark gather (k_lm_gather*), of k_sb_elim (the graph runs it beside the gather) and of the
    reprojection kernel k_proj_lin_pp (the writer of the landmark records);
  - how much of the gather's time runs beside k_sb_elim;
  - the record and Wt bytes the gather moves, computed from the shapes (records read, the scaled coupling rows Wt
    written: nl x ldw doubles per window), and the resulting GB/s over the gather's time.

    python tools/gather_probe.py --out DIR [--batch 528] [--iters 8]

The record width is taken from the gather kernel in the trace (k_lm_gather12: 12 doubles, k_lm_gather16: 16).  The
trace goes to DIR/gather.pt.trace.json and the summary to DIR/gather.json (also printed).  The tree the script sits in
is the one imported, so a copy of the script inside another checkout measures that checkout.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def merge(iv):
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def overlap(a, b, merged):
    return sum(max(0.0, min(b, y) - max(a, x)) for x, y in merged)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=528)
    ap.add_argument("--iters", type=int, default=8)
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from d2slam_b200 import abi
    from d2slam_b200.solver import Solver

    if not torch.cuda.is_available():
        sys.exit("gather_probe: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    probs = bench.make_batch(args.batch, 1000)
    s = Solver(max_windows=args.batch, max_num_iterations=args.iters)
    bench.load_all(s, probs)
    s.finalize()
    for _ in range(3):   # the iteration graph is captured from the second solve on
        bench.reset_state(s, probs)
        s.solve_fixed(args.iters)
    torch.cuda.synchronize()
    bench.reset_state(s, probs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.solve_fixed(args.iters)
        torch.cuda.synchronize()
    trace = os.path.join(args.out, "gather.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])

    def short(n):
        n = n.split("(")[0].split("<")[0]
        return n.replace("void ", "").replace("d2ba::", "").strip()

    k = [(short(e["name"]), float(e["ts"]), float(e["ts"]) + float(e["dur"])) for e in ev]
    n_ctl = sum(1 for n, *_ in k if n == "k_control")
    per = {}
    for n, a, b in k:
        d = per.setdefault(n, [0, 0.0])
        d[0] += 1
        d[1] += b - a
    gathers = sorted(n for n in per if n.startswith("k_lm_gather"))
    watch = gathers + sorted(n for n in per if n == "k_sb_elim" or n.startswith("k_proj_lin"))
    sbe = merge([[a, b] for n, a, b in k if n == "k_sb_elim"])
    g_us = sum(b - a for n, a, b in k if n in gathers)
    g_beside = sum(overlap(a, b, sbe) for n, a, b in k if n in gathers)
    # bytes from the shapes: one record per residual, one Wt row of ldw = roundup(n_lc + 1, 8) doubles per landmark
    rec_doubles = 12 if "k_lm_gather12" in per else 16
    n_res = sum(int(p["obs"].shape[0]) for p in probs)
    wt_doubles = 0
    for i, p in enumerate(probs):
        nlc = int(np.asarray(s.debug_get(i, abi.DBG_N_LC, np.int64)).reshape(-1)[0])
        wt_doubles += len(p["lm_ids"]) * ((nlc + 1 + 7) // 8 * 8)
    rec_bytes = n_res * rec_doubles * 8
    wt_bytes = wt_doubles * 8
    n_g = max(1, max((per[n][0] for n in gathers), default=0))   # gather launches (the kernels of one iteration share it)
    g_us_it = g_us / n_g
    res = {
        "gpu": torch.cuda.get_device_name(0),
        "batch": args.batch, "iters": args.iters, "k_control_launches": n_ctl,
        "kernel_us_per_launch": {n: round(per[n][1] / per[n][0], 2) for n in watch},
        "launches": {n: per[n][0] for n in watch},
        "gather_us_per_iteration": round(g_us_it, 2),
        "gather_beside_sb_elim_us_per_iteration": round(g_beside / n_g, 2),
        "gather_beside_sb_elim_fraction": round(g_beside / g_us, 3) if g_us > 0 else None,
        "record_doubles": rec_doubles,
        "record_bytes_per_iteration": rec_bytes,
        "wt_bytes_per_iteration": wt_bytes,
        "gather_gbs": round((rec_bytes + wt_bytes) / (g_us_it * 1e-6) / 1e9, 1) if g_us_it > 0 else None,
        "kernel_ms_per_iteration": {n: round(v, 5) for n, v in s.kernel_times(args.iters).items()},
    }
    with open(os.path.join(args.out, "gather.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
