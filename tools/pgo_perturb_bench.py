"""Pose-graph chart benchmark: the bench's 6-DoF pose graph solved in d2pgo's perturbation chart (PgoSolver.set_chart("perturb"):
states [p, theta], q = q_init (x) quatfromRotationVector(theta)) beside the retraction chart, both from the same initial poses,
under ceres' Levenberg-Marquardt at d2pgo's defaults (50 iterations, no time budget) and under the restated LM loop, all with
exact steps from the sparse Cholesky.

Workload: pgo.make_pose_graph(seed=7): 8 agents x 1250 poses, 40 000 edges; optionally one gravity prior per pose
(--gravity).  Per minimiser and chart, after one warm-up, `--solves` solves from a fresh handle, alternating.  Prints one JSON
line: the card and its power limit; per minimiser and chart the iterations (successful / unsuccessful), the termination and
stop reason, median device ms and ms per iteration, the final cost; per minimiser the largest position / attitude difference
between the two charts' results (d2pgo_get_poses).  Writes nothing.

    python tools/pgo_perturb_bench.py [--solves 3] [--gravity]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo  # noqa: E402
from pgo_4dof_bench import card  # noqa: E402
from pgo_cholesky_bench import CHOLESKY, pose_diff  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=3, help="timed solves per minimiser and chart after one warm-up each (median reported)")
    ap.add_argument("--gravity", action="store_true", help="one gravity prior per pose (pgo.make_gravity_case)")
    args = ap.parse_args()
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    ego = pgo.make_gravity_case(g, seed=7)["ego"] if args.gravity else None
    N = len(g["ids"])

    def make(minimizer, chart):
        s = pgo.PgoSolver(**CHOLESKY)
        if minimizer == "ceres_lm":
            s.set_minimizer("ceres_lm")
        s.set_poses(g["ids"], g["init"], g["fixed"])
        if chart == "perturb":
            s.set_chart("perturb")
        s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
        if ego is not None:
            s.add_gravity_priors(g["ids"], ego)
        return s

    out = {"metric": "pgo_perturb_chart", "card": card(),
           "workload": f"{N} poses / {len(g['id_a'])} edges{' + one gravity prior per pose' if ego is not None else ''}, 1 GPU",
           "settings": {"ceres_lm": "ceres defaults (d2pgo's LEVENBERG_MARQUARDT)", "restated": CHOLESKY}, "solves": args.solves, "minimizers": {}}
    charts = ("retraction", "perturb")
    for minimizer in ("ceres_lm", "restated"):
        for chart in charts:   # warm-up: module load, analysis, graph capture
            s = make(minimizer, chart); s.solve(); s.close()
        runs = {c: [] for c in charts}
        last = {}
        for _ in range(args.solves):
            for chart in charts:
                s = make(minimizer, chart)
                r = s.solve()
                rep = s.minimizer_report() if minimizer == "ceres_lm" else None
                last[chart] = (r, rep, s.get_poses(g["ids"]))
                runs[chart].append(r.device_ms)
                s.close()
        res = {}
        for chart in charts:
            r, rep, _ = last[chart]
            ms = float(np.median(runs[chart]))
            leg = {"iterations": r.iterations, "successful": r.accepted, "unsuccessful": r.iterations - r.accepted,
                   "device_ms_median": ms, "device_ms_all": [round(m, 3) for m in runs[chart]], "ms_per_iteration": ms / max(1, r.iterations),
                   "initial_cost": r.initial_cost, "final_cost": r.final_cost}
            if rep is not None:
                leg.update(termination=rep["termination"], stop=rep["stop"])
            res[chart] = leg
        dp, dr = pose_diff(last["perturb"][2], last["retraction"][2])
        res["max_position_diff_between_charts_m"] = dp
        res["max_attitude_diff_between_charts_rad"] = dr
        out["minimizers"][minimizer] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
