"""Pose-graph minimiser benchmark: ceres' Levenberg-Marquardt trust region decided on the device (PgoSolver.set_minimizer(
"ceres_lm"), d2pgo's LEVENBERG_MARQUARDT) beside the restated LM loop, both with exact steps from the sparse Cholesky, on the same
graphs in the same call.

Workload: the bench's pose graph (pgo.make_pose_graph(seed=7): 8 agents x 1250 poses, 40 000 edges) as 6-DoF, as 4-DoF
(pgo.pose_graph_to_4d) and as 6-DoF with one gravity prior per pose (pgo.make_gravity_case).  Per graph, after one warm-up each,
`--solves` solves of each minimiser from the initial poses, alternating.  Prints one JSON line: the card and its power limit;
per graph and minimiser the successful / unsuccessful iterations and the termination, median device ms and ms per iteration,
host synchronisations per solve (ceres: the minimiser's report, which counts the uploads of the fresh handle's graph and
factor tables; restated: one
per linearisation and one per factorisation, 2 + 2 iterations - failed factorisations, plus the two uploads'), the final cost against
the CPU oracle's converged cost (scipy sparse direct Gauss-Newton, run until the relative cost change is below 1e-13) and the
largest position / attitude difference to the oracle's optimum.  Writes nothing.

    python tools/pgo_ceres_lm_bench.py [--solves 5] [--oracle-iters 40]
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

CERES = {}   # ceres' defaults (max_num_iterations 50, function_tolerance 1e-6, no time budget)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=5, help="timed solves per minimiser after one warm-up each (median reported)")
    ap.add_argument("--oracle-iters", type=int, default=40, help="most Gauss-Newton iterations of the CPU oracle (it stops earlier once converged)")
    args = ap.parse_args()
    from oracle import pgo4d_oracle as p4
    from oracle import pgo_gravity_oracle as go
    from oracle import pgo_oracle as po
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    h = pgo.pose_graph_to_4d(g, seed=7)
    c = pgo.make_gravity_case(g, seed=7)
    N = len(g["ids"])
    idx = np.arange(N); u_ego = go.ego_gravity(c["ego"]); S = np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (N, 1, 1))
    graphs = {
        "6dof": (g, 6, None, lambda: po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=args.oracle_iters, ftol=1e-13),
                 lambda x: go.cost_gravity(x, g["ea"], g["eb"], g["rel"], g["sqrt_info"], [], np.zeros((0, 3)), np.zeros((0, 3, 3)))),
        "4dof": (h, 4, None, lambda: p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"], iters=args.oracle_iters, ftol=1e-13),
                 lambda x: p4.cost_4d(x, h["ea"], h["eb"], h["rel"], h["sqrt_info"])),
        "6dof_gravity": (g, 6, c["ego"], lambda: go.solve_gravity(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S,
                                                                  iters=args.oracle_iters, ftol=1e-13),
                         lambda x: go.cost_gravity(x, g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)),
    }
    out = {"metric": "pgo_ceres_lm", "card": card(),
           "workload": f"{N} poses / {len(g['id_a'])} edges (8 trajectories, odometry + loop closures), 1 GPU",
           "settings": {"ceres_lm": CERES or "ceres defaults", "restated": CHOLESKY}, "solves": args.solves, "graphs": {}}
    for name, (gr, dof, ego, oracle_solve, oracle_cost) in graphs.items():
        def make(kind):
            s = pgo.PgoSolver(pose_dof=dof, **CHOLESKY)
            if kind == "ceres_lm":
                s.set_minimizer("ceres_lm", **CERES)
            if dof == 4:
                s.set_poses_4d(gr["ids"], gr["init"], gr["fixed"]); s.add_edges_4d(gr["id_a"], gr["id_b"], gr["rel"], gr["sqrt_info"])
            else:
                s.set_poses(gr["ids"], gr["init"], gr["fixed"]); s.add_edges(gr["id_a"], gr["id_b"], gr["rel"], gr["sqrt_info"])
                if ego is not None:
                    s.add_gravity_priors(gr["ids"], ego)
            return s
        kinds = ("ceres_lm", "restated")
        runs = {k: [] for k in kinds}
        last = {}
        for kind in kinds:   # warm-up: module load, analysis, graph capture
            s = make(kind); s.solve(); s.close()
        for _ in range(args.solves):
            for kind in kinds:
                s = make(kind)
                r = s.solve()
                st = s.cholesky_stats()
                rep = s.minimizer_report() if kind == "ceres_lm" else None
                x = s.get_poses_4d(gr["ids"]) if dof == 4 else s.get_poses(gr["ids"])
                s.close()
                runs[kind].append(r); last[kind] = (r, st, rep, x)
        xr, costs = oracle_solve()
        ref = oracle_cost(xr)
        res = {"oracle_converged_cost": ref, "oracle_iterations": len(costs),
               "oracle_last_rel_cost_change": abs(costs[-2] - costs[-1]) / costs[-1] if len(costs) > 1 else None}
        for kind in kinds:
            r, st, rep, x = last[kind]
            ms = [q.device_ms for q in runs[kind]]
            dp, dr = pose_diff(x, xr)
            leg = {"iterations": r.iterations, "successful": r.accepted, "unsuccessful": r.iterations - r.accepted, "converged": int(r.converged),
                   "device_ms_median": float(np.median(ms)), "device_ms_all": [round(m, 3) for m in ms],
                   "ms_per_iteration": float(np.median(ms)) / max(1, r.iterations), "final_cost": r.final_cost,
                   "cost_rel_diff_vs_oracle": (r.final_cost - ref) / ref, "max_position_diff_vs_oracle_m": dp, "max_attitude_diff_vs_oracle_rad": dr}
            if rep is not None:
                leg.update(termination=rep["termination"], stop=rep["stop"], host_syncs=rep["host_syncs"], elapsed_device_s=rep["elapsed_s"],
                           final_radius=rep["final_radius"])
            else:
                # one per linearisation and factorisation and the final read, plus the uploads of the graph and of the factor's tables
                leg["host_syncs"] = 2 + 2 * r.iterations - st["failed_factorizations"] + 2
            res[kind] = leg
        out["graphs"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
