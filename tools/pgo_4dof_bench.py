"""4-DoF pose-graph benchmark (d2pgo's default RelPoseFactor4D configuration) beside the 6-DoF solve of the same graph.

Workload: the bench's pose-graph graph (pgo.make_pose_graph(seed=7): 8 agents x 1250 poses, 40 000 edges) through
pgo.pose_graph_to_4d, solved with bench.py pgo_leg's settings (inexact LM + block-Jacobi PCG).  Prints one JSON line: the card
and its power limit, median device_ms of the timed solves after one warm-up, LM / PCG iterations, the 6-DoF numbers of the
same graph, the CPU oracle's time and converged cost (oracle/pgo4d_oracle.py, scipy sparse direct) and the device solution's
position / yaw error against the oracle's.  Writes nothing.

    python tools/pgo_4dof_bench.py [--solves 5] [--oracle-iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo, synth  # noqa: E402

SETTINGS = dict(max_iterations=60, pcg_max_iterations=200, pcg_tolerance=1e-1, lambda0=1e-4, function_tolerance=1e-5)   # bench.py pgo_leg


def card(index=0):
    """Card name and power limit (read-only nvidia-smi query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def timed(make, n):
    s = make()
    s.solve()                                     # warm-up: module load, graph capture
    reps = []
    for _ in range(n):
        s.close(); s = make()
        reps.append(s.solve())
    return s, reps


def summary(reps):
    ms = [r.device_ms for r in reps]
    r = reps[-1]
    return {"device_ms_median": float(np.median(ms)), "device_ms_all": [round(m, 3) for m in ms], "lm_iterations": r.iterations,
            "pcg_iterations": r.pcg_iterations, "initial_cost": r.initial_cost, "final_cost": r.final_cost, "converged": int(r.converged)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=5, help="timed solves after the warm-up (median reported)")
    ap.add_argument("--oracle-iters", type=int, default=10, help="Gauss-Newton iterations of the CPU oracle")
    args = ap.parse_args()
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)   # + 7 connecting closures = 40 000 edges
    h = pgo.pose_graph_to_4d(g, seed=7)

    def make4():
        s = pgo.PgoSolver(pose_dof=4, **SETTINGS)
        s.set_poses_4d(h["ids"], h["init"], h["fixed"]); s.add_edges_4d(h["id_a"], h["id_b"], h["rel"], h["sqrt_info"])
        return s

    def make6():
        s = pgo.PgoSolver(**SETTINGS)
        s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
        return s
    s4, reps4 = timed(make4, args.solves)
    x4 = s4.get_poses_4d(h["ids"]); s4.close()
    s6, reps6 = timed(make6, args.solves)
    x6 = s6.get_poses(g["ids"]); s6.close()

    from oracle import pgo4d_oracle as p4
    t0 = time.perf_counter()
    x_ref, costs = p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"], iters=args.oracle_iters)
    dt = time.perf_counter() - t0
    final_ref = p4.cost_4d(x_ref, h["ea"], h["eb"], h["rel"], h["sqrt_info"])
    err = lambda x, y: (float(np.linalg.norm(x[:, :3] - y[:, :3], axis=1).max()), float(np.abs(pgo.normalize_angle(x[:, 3] - y[:, 3])).max()))
    dp, dyaw = err(x4, x_ref)
    out = {"metric": "pgo_4dof", "card": card(),
           "workload": f"{len(h['ids'])} poses / {len(h['id_a'])} edges (8 trajectories, odometry + loop closures), RelPoseFactor4D on [x y z yaw], "
                       "inexact LM + block-Jacobi PCG (bench.py pgo_leg settings), 1 GPU",
           "settings": SETTINGS, "solves": args.solves,
           "dof4": summary(reps4), "dof6_same_graph": summary(reps6),
           "max_position_error_vs_ground_truth_m": {"dof4_initial_guess": err(h["init"], h["gt"])[0], "dof4_solved": err(x4, h["gt"])[0],
                                                    "dof4_oracle_solved": err(x_ref, h["gt"])[0], "dof6_solved": float(synth.pose_errors(x6, g["gt"])[0])},
           "cpu_oracle_4dof": {"what": "numpy linearisation + scipy sparse direct Gauss-Newton (oracle/pgo4d_oracle.py), 1 process",
                               "iterations": len(costs), "seconds": dt, "converged_cost": final_ref},
           "dof4_vs_oracle": {"max_position_diff_m": dp, "max_yaw_diff_rad": dyaw, "cost_rel_diff": (reps4[-1].final_cost - final_ref) / final_ref}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
