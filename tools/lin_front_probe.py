"""Where the linearisation front of the bench workload spends its time.

Runs the flagship workload of bench.py (make_batch(528, 1000), 8 fixed iterations, device-resident solve_fixed), takes
one torch.profiler trace (CUDA activities) of a CUDA-graph replay and reports:
  - per-kernel device time of k_misc_lin and the IMU kernels (k_imu*), and of the reprojection kernel k_proj_lin_pp;
  - how much of each IMU kernel's time runs beside k_proj_lin_pp / k_misc_lin (the graph's two lanes);
  - the span of the linearisation front per iteration (start of k_misc_lin to the end of the last IMU / reprojection
    kernel before k_control);
  - the kernel_times buckets (CUDA events around each stage, serial, no graph).

    python tools/lin_front_probe.py --out DIR [--batch 528] [--iters 8]

The trace goes to DIR/lin_front.pt.trace.json and the summary to DIR/lin_front.json (also printed).  The tree the script
sits in is the one imported, so a copy of the script inside another checkout measures that checkout.
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
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from d2slam_b200.solver import Solver

    if not torch.cuda.is_available():
        sys.exit("lin_front_probe: no CUDA device")
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
    trace = os.path.join(args.out, "lin_front.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])

    def short(n):
        n = n.split("(")[0].split("<")[0]
        return n.replace("void ", "").replace("d2ba::", "").strip()

    k = [(short(e["name"]), float(e["ts"]), float(e["ts"]) + float(e["dur"]), e["args"].get("stream")) for e in ev]
    n_iter = sum(1 for n, *_ in k if n == "k_control")
    per = {}
    for n, a, b, _ in k:
        d = per.setdefault(n, [0, 0.0])
        d[0] += 1
        d[1] += b - a
    watch = sorted(n for n in per if n == "k_misc_lin" or n.startswith("k_imu") or n.startswith("k_proj_lin"))
    pp = merge([[a, b] for n, a, b, _ in k if n.startswith("k_proj_lin")])
    ml = merge([[a, b] for n, a, b, _ in k if n == "k_misc_lin"])
    side = {}
    for n in watch:
        if not n.startswith("k_imu"):
            continue
        tot = sum(b - a for m, a, b, _ in k if m == n)
        ov_pp = sum(overlap(a, b, pp) for m, a, b, _ in k if m == n)
        ov_ml = sum(overlap(a, b, ml) for m, a, b, _ in k if m == n)
        side[n] = {"us_total": round(tot, 2), "beside_proj_lin_us": round(ov_pp, 2), "beside_misc_lin_us": round(ov_ml, 2),
                   "hidden_fraction": round((ov_pp + ov_ml) / tot, 3) if tot > 0 else None}
    # linearisation front per iteration: from each k_misc_lin start to the end of the last front kernel before k_control
    fronts = []
    for n, a, _, _ in k:
        if n != "k_misc_lin":
            continue
        end = a
        for m, x, y, _ in k:
            if x < a:
                continue
            if m == "k_control":
                break
            if m.startswith("k_imu") or m.startswith("k_proj_lin") or m == "k_misc_lin":
                end = max(end, y)
        fronts.append(end - a)
    span = (k[-1][2] - k[0][1]) if k else 0.0
    kt = s.kernel_times(args.iters)
    res = {
        "gpu": torch.cuda.get_device_name(0),
        "batch": args.batch, "iters": args.iters, "graph_iterations_traced": n_iter,
        "kernel_us_per_iteration": {n: round(per[n][1] / max(1, n_iter), 2) for n in watch},
        "launches_per_iteration": {n: per[n][0] / max(1, n_iter) for n in watch},
        "imu_overlap_us_per_solve": side,
        "front_span_us_per_iteration": round(sum(fronts) / max(1, len(fronts)), 2),
        "trace_span_us": round(span, 1),
        "kernel_ms_per_iteration": {n: round(v, 5) for n, v in kt.items()},
    }
    with open(os.path.join(args.out, "lin_front.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
