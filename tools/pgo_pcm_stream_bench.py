"""PCM as a stream (d2pgo_pcm_stream) on the bench pose graph of tools/pgo_pcm_bench.py (make_pose_graph seed 7, 5 % injected
gross outliers, pcm_thres 3.5, covariance rates 0.5 / 1e-2), revealed in --steps arrival steps (pgo.pcm_arrival_steps; each
call passes every loop so far, as D2PGO does).  Per pose dof and clique mode: device time per call (median, p90, max), the
pair and clique parts, pairs tested; then one d2pgo_pcm on the final input in the same process.  Mode 0's final mask is
compared bitwise with that batch; both modes report recall and precision of the rejection against the injected outliers.
The card's name and power limit are read in the same run.

    python tools/pgo_pcm_stream_bench.py [--dof 4 6] [--steps 100] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo  # noqa: E402
from pgo_pcm_bench import card  # noqa: E402


def quality(mask, outlier):
    rej = ~mask
    return dict(recall=float((rej & outlier).sum() / max(outlier.sum(), 1)), precision=float((rej & outlier).sum() / max(rej.sum(), 1)),
                inliers=int(mask.sum()))


def run_stream(s, c, steps, incremental, cfg):
    s.pcm_stream_reset(incremental, **cfg)
    seen = np.zeros(0, np.int64); per = []
    for f, l in steps:
        seen = np.concatenate([seen, l])
        mask = s.pcm_stream(*pgo.pcm_stream_args(c, f, seen)); r = s.pcm_stream_report
        per.append((r.device_ms, r.pair_ms, r.clique_ms, r.new_loops, r.groups_touched, r.pairs_tested, r.clique_rounds))
    a = np.array(per)
    dev = a[:, 0]
    return mask, seen, dict(mode=incremental, calls=len(per), device_ms_median=float(np.median(dev)), device_ms_p90=float(np.percentile(dev, 90)),
                            device_ms_max=float(dev.max()), device_ms_total=float(dev.sum()), pair_ms_total=float(a[:, 1].sum()),
                            clique_ms_total=float(a[:, 2].sum()), pair_ms_median=float(np.median(a[:, 1])), clique_ms_median=float(np.median(a[:, 2])),
                            pairs_tested=int(a[:, 5].sum()), clique_rounds=int(a[:, 6].sum()), device_ms_per_call=dev.tolist(),
                            new_loops_per_call=a[:, 3].astype(int).tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dof", type=int, nargs="+", default=[4, 6], choices=(4, 6))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out")
    a = ap.parse_args()
    g = pgo.make_pose_graph(seed=7)
    c = pgo.make_pcm_case(g, 0.05, seed=7)
    cfg = dict(pcm_thres=3.5, pos_covariance_per_meter=0.5, yaw_covariance_per_meter=1e-2)
    steps = pgo.pcm_arrival_steps(c, a.steps)
    name, pl = card()
    res = dict(workload="make_pose_graph seed 7, 5% outliers, streamed", steps=a.steps, loops=int(len(c["kf_a"])), config=cfg, card=name, power_limit=pl,
               runs=[])
    for dof in a.dof:
        s = pgo.PgoSolver(pose_dof=dof)
        run_stream(s, c, pgo.pcm_arrival_steps(c, 5)[:2], 0, cfg)   # warm-up: module load, first allocations
        out = dict(pose_dof=dof)
        for inc in (0, 1):
            mask, order, st = run_stream(s, c, steps, inc, cfg)
            st.update(quality(mask, c["outlier"][order]))
            out[f"mode{inc}"] = st
            if inc == 0:
                final0 = mask
        args = (c["frame_ids"], c["frame_agent"], c["ego"], c["kf_a"][order], c["kf_b"][order], c["rel_bad"][order], c["sqrt_info"][order])
        s.pcm(*args, **cfg)   # warm-up of the batch's buffers
        bm = s.pcm(*args, **cfg); r = s.pcm_report
        out["batch"] = dict(device_ms=r.device_ms, pair_ms=r.pair_ms, clique_ms=r.clique_ms, pairs_tested=int(r.pairs_tested), **quality(bm, c["outlier"][order]))
        out["mode0_final_mask_equals_batch"] = bool(np.array_equal(final0, bm))
        res["runs"].append(out)
        print(json.dumps({k: (v if not isinstance(v, dict) else {kk: vv for kk, vv in v.items() if not kk.endswith("per_call")}) for k, v in out.items()}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
