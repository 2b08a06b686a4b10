"""Gravity-prior pose-graph benchmark (d2pgo's 6-DoF configuration with enable_gravity_prior) beside the same solve without priors.

Workload: the bench's pose-graph graph (pgo.make_pose_graph(seed=7): 8 agents x 1250 poses, 40 000 edges), 6-DoF, one gravity
prior on every pose (ego poses from pgo.make_gravity_case, S = gravity_sqrt_info I3 = 10 I3), solved with bench.py pgo_leg's
settings (inexact LM + block-Jacobi PCG).  Prints one JSON line: the card and its power limit; with and without priors the
median device_ms of the timed solves after one warm-up, LM / PCG iterations, the final cost against the CPU oracle's converged
cost of the same problem (oracle/pgo_gravity_oracle.py, oracle/pgo_oracle.py) and the roll / pitch RMS error to ground truth.
Writes nothing.

    python tools/pgo_gravity_bench.py [--solves 5] [--oracle-iters 10]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo  # noqa: E402
from pgo_4dof_bench import SETTINGS, card, summary, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=5, help="timed solves after the warm-up (median reported)")
    ap.add_argument("--oracle-iters", type=int, default=10, help="Gauss-Newton iterations of the CPU oracle")
    args = ap.parse_args()
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)   # + 7 connecting closures = 40 000 edges
    c = pgo.make_gravity_case(g, seed=7)
    N = len(g["ids"])

    def make(priors):
        def f():
            s = pgo.PgoSolver(**SETTINGS)
            s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
            if priors:
                s.add_gravity_priors(g["ids"], c["ego"])
            return s
        return f
    sg, reps_g = timed(make(True), args.solves)
    xg = sg.get_poses(g["ids"]); sg.close()
    s0, reps_0 = timed(make(False), args.solves)
    x0 = s0.get_poses(g["ids"]); s0.close()

    from oracle import pgo_gravity_oracle as go
    from oracle import pgo_oracle as po
    idx = np.arange(N); u_ego = go.ego_gravity(c["ego"]); S = np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (N, 1, 1))
    xr_g, costs_g = go.solve_gravity(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S, iters=args.oracle_iters)
    xr_0, costs_0 = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=args.oracle_iters)
    ref_g = go.cost_gravity(xr_g, g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)
    ref_0 = go.cost_gravity(xr_0, g["ea"], g["eb"], g["rel"], g["sqrt_info"], [], np.zeros((0, 3)), np.zeros((0, 3, 3)))
    rms = lambda x: float(np.degrees(np.sqrt(np.mean(go.tilt_errors(x, g["gt"]) ** 2))))

    def leg(reps, x, ref_cost, xr):
        out = summary(reps)
        out.update({"oracle_converged_cost": ref_cost, "cost_rel_diff_vs_oracle": (reps[-1].final_cost - ref_cost) / ref_cost,
                    "roll_pitch_rms_error_deg": rms(x), "oracle_roll_pitch_rms_error_deg": rms(xr)})
        return out
    out = {"metric": "pgo_gravity_prior", "card": card(),
           "workload": f"{N} poses / {len(g['id_a'])} edges (8 trajectories, odometry + loop closures) + {N} gravity priors (S = 10 I3), "
                       "6-DoF RelPoseFactorAD + GravityPriorPerturbAD, inexact LM + block-Jacobi PCG (bench.py pgo_leg settings), 1 GPU",
           "settings": SETTINGS, "solves": args.solves,
           "with_priors": leg(reps_g, xg, ref_g, xr_g), "without_priors": leg(reps_0, x0, ref_0, xr_0),
           "roll_pitch_rms_error_deg_initial_guess": rms(g["init"]), "roll_pitch_rms_error_deg_ego_poses": rms(c["ego"]),
           "oracle": {"what": "numpy linearisation + scipy sparse direct Gauss-Newton, 1 process", "iterations": [len(costs_g), len(costs_0)]}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
