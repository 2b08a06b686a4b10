"""PCM loop-closure outlier rejection on the bench pose graph (make_pose_graph seed 7: 8 drones, 10 000 poses, 30 000 loops)
with 5 % injected gross outliers: median device time of five d2pgo_pcm calls and its pair / clique split, pairs tested per
second, clique rounds, precision and recall of the rejection against the injected outliers, and the card it ran on.
--ref adds the reference's own PCM (oracle/_ref/libd2ref_pcm.so, one host thread) for context, labelled as a CPU time.

    python tools/pgo_pcm_bench.py [--dof 4|6] [--ref] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[0]
        name, pl = [x.strip() for x in q.split(",")]
        return name, pl
    except Exception as e:   # the card name is part of the number; say so when it cannot be read
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dof", type=int, default=4, choices=(4, 6))
    ap.add_argument("--thres", type=float, default=3.5)
    ap.add_argument("--pos-cov", type=float, default=0.5)
    ap.add_argument("--yaw-cov", type=float, default=1e-2)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--ref", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    g = pgo.make_pose_graph(seed=7)
    c = pgo.make_pcm_case(g, 0.05, seed=7)
    cfg = dict(pcm_thres=a.thres, pos_covariance_per_meter=a.pos_cov, yaw_covariance_per_meter=a.yaw_cov)
    s = pgo.PgoSolver(pose_dof=a.dof)
    args = (c["frame_ids"], c["frame_agent"], c["ego"], c["kf_a"], c["kf_b"], c["rel_bad"], c["sqrt_info"])
    mask = s.pcm(*args, **cfg)   # warm-up: module load, allocations
    reps, masks = [], []
    for _ in range(a.calls):
        masks.append(s.pcm(*args, **cfg)); r = s.pcm_report
        reps.append((r.device_ms, r.pair_ms, r.clique_ms))
    assert all(np.array_equal(m, mask) for m in masks)
    r = s.pcm_report
    k = int(np.argsort([x[0] for x in reps])[len(reps) // 2])
    dev_ms, pair_ms, clique_ms = reps[k]
    rejected = ~mask; out = c["outlier"]
    name, pl = card()
    res = dict(workload="make_pose_graph seed 7, 5% outliers", pose_dof=a.dof, loops=int(len(mask)), groups=r.groups, pairs_tested=int(r.pairs_tested),
               consistent_pairs=int(r.consistent_pairs), clique_rounds=int(r.clique_rounds), inliers=r.inliers,
               device_ms_median=dev_ms, pair_ms=pair_ms, clique_ms=clique_ms, pairs_per_s=r.pairs_tested / (pair_ms * 1e-3),
               precision=float((rejected & out).sum() / max(rejected.sum(), 1)), recall=float((rejected & out).sum() / max(out.sum(), 1)),
               device_ms_all=[x[0] for x in reps], card=name, power_limit=pl, config=cfg)
    if a.ref:
        from oracle import ref_pcm as ref
        t = time.perf_counter()
        good, _ = ref.pcm(c, a.dof == 4, a.thres, a.pos_cov, a.yaw_cov, rel_key="rel_bad")
        res["reference_cpu_ms_one_thread"] = (time.perf_counter() - t) * 1e3
        res["reference_mask_equal"] = bool(np.array_equal(good, mask))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
