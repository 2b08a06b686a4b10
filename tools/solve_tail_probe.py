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
  - the CTAs per SM of k_solve_small (cudaOccupancyMaxActiveBlocksPerMultiprocessor at the handle's shared memory).

    python tools/solve_tail_probe.py --out DIR [--batch 528] [--iters 8]

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


def tail_bytes(s, probs):
    import numpy as np
    from d2slam_b200 import abi
    total = 0
    for i, p in enumerate(probs):
        nlc = int(np.asarray(s.debug_get(i, abi.DBG_N_LC, np.int64)).reshape(-1)[0])
        n_c = int(np.asarray(s.debug_get(i, abi.DBG_N_CAM, np.int64)).reshape(-1)[0])
        nl, nb = len(p["lm_ids"]), (n_c - nlc) // 9
        ldw = (nlc + 1 + 7) // 8 * 8
        wt_rows = (nl + 9 * nb + 31) // 32 * 32
        total += (wt_rows * ldw + 9 * nb * (nlc + 1) + 171 * nb + nl * ldw) * 8
    return total


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
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=528)
    ap.add_argument("--iters", type=int, default=8)
    args = ap.parse_args()
    import torch
    import bench

    if not torch.cuda.is_available():
        sys.exit("solve_tail_probe: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    probs = bench.make_batch(args.batch, 1000)
    res = {"gpu": torch.cuda.get_device_name(0), "batch": args.batch, "iters": args.iters}
    for path in ("separate", "fused"):
        res[path] = run(path, args, probs)
    a, b = res["separate"]["tail_span_us_per_iteration"], res["fused"]["tail_span_us_per_iteration"]
    res["fused_over_separate_span"] = round(b / a, 3) if a and b else None
    with open(os.path.join(args.out, "solve_tail.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
