"""Chordal rotation initialisation benchmark (include/d2pgo.h d2pgo_rot_init; d2pgo's rotInitial) and its effect on the 6-DoF
solve that follows.

Workload: the bench's pose-graph graph (pgo.make_pose_graph(seed=7): 8 agents x 1250 poses, 40 000 edges), 6-DoF, pose 0
fixed.  Prints one JSON line with the card and its power limit and, without and with gravity rows (ego poses from
pgo.make_gravity_case, g = 10):
  - rot init: median device_ms of the timed calls after one warm-up, CG iterations and the relative residual reached per row
    system, the rotation RMS error to the ground truth before and after, and the largest rotation difference to the CPU oracle's
    rot init (oracle/pgo_rotinit_oracle.py, scipy sparse direct) with the oracle's host time;
  - bench.py pgo_leg's inexact-LM solve from the raw initial guess and from the rot-init guess (with gravity rows: both with
    d2pgo_add_gravity_priors): LM / PCG counts, device ms, final cost against the oracle's converged cost, largest position /
    rotation error to the oracle's converged poses and to the ground truth.
Writes nothing.

    python tools/pgo_rotinit_bench.py [--calls 5] [--oracle-iters 10]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo, synth  # noqa: E402
from pgo_4dof_bench import SETTINGS, card, summary  # noqa: E402


def rot_rms_deg(x, gt):
    from oracle import pgo_rotinit_oracle as ro
    R, G = ro.quat_R(np.asarray(x)[:, 3:7]), ro.quat_R(np.asarray(gt)[:, 3:7])
    c = np.clip((np.einsum("nij,nij->n", R, G) - 1.0) / 2.0, -1.0, 1.0)
    return float(np.degrees(np.sqrt(np.mean(np.arccos(c) ** 2))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5, help="timed rot-init calls and solves after the warm-up (median reported)")
    ap.add_argument("--oracle-iters", type=int, default=10, help="Gauss-Newton iterations of the CPU oracle's converged solve")
    args = ap.parse_args()
    from oracle import pgo_gravity_oracle as go
    from oracle import pgo_oracle as po
    from oracle import pgo_rotinit_oracle as ro
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)   # + 7 connecting closures = 40 000 edges
    c = pgo.make_gravity_case(g, seed=7)
    N = len(g["ids"])
    idx = np.arange(N); u_ego = go.ego_gravity(c["ego"]); S = np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (N, 1, 1))

    def handle(priors, **kw):
        s = pgo.PgoSolver(**kw)
        s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
        if priors:
            s.add_gravity_priors(g["ids"], c["ego"])
        return s

    def rot_init(s, grav):
        return s.rot_init(g["ids"], c["ego"], enable_gravity_prior=1) if grav else s.rot_init()

    xr = {}
    t0 = time.perf_counter(); xr[False], costs0 = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=args.oracle_iters)
    t_or0 = time.perf_counter() - t0
    xr[True], costsg = go.solve_gravity(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S, iters=args.oracle_iters)
    ref_cost = {False: go.cost_gravity(xr[False], g["ea"], g["eb"], g["rel"], g["sqrt_info"], [], np.zeros((0, 3)), np.zeros((0, 3, 3))),
                True: go.cost_gravity(xr[True], g["ea"], g["eb"], g["rel"], g["sqrt_info"], idx, u_ego, S)}

    out = {"metric": "pgo_rot_init", "card": card(),
           "workload": f"{N} poses / {len(g['id_a'])} edges (8 trajectories, odometry + loop closures), 6-DoF, pose 0 fixed; "
                       "rot init then bench.py pgo_leg's inexact LM + block-Jacobi PCG, 1 GPU",
           "settings": SETTINGS, "calls": args.calls, "rot_rms_error_deg_initial_guess": rot_rms_deg(g["init"], g["gt"]),
           "oracle_converged_solve_s": t_or0}
    for grav in (False, True):
        leg = {}
        s = handle(False)
        rot_init(s, grav)                                  # warm-up: module load, allocation, graph capture
        reps = []
        for _ in range(args.calls):
            s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
            reps.append(rot_init(s, grav))
        x_ri = s.get_poses(g["ids"]); s.close()
        t0 = time.perf_counter()
        o = ro.rot_init(g["ids"], g["init"], g["fixed"], g["id_a"], g["id_b"], g["rel"], g["sqrt_info"], gravity=grav, ego_ids=g["ids"], ego_poses=c["ego"])
        t_or = time.perf_counter() - t0
        rows = np.searchsorted(g["ids"], np.asarray(o["frames"], np.int64))
        r = reps[-1]
        dR = np.abs(ro.quat_R(x_ri[rows, 3:7]) - o["R"]).max(axis=(1, 2)); worst = int(np.argmax(dR))
        leg["rot_init"] = {"device_ms_median": float(np.median([q["device_ms"] for q in reps])), "device_ms_all": [round(q["device_ms"], 3) for q in reps],
                           "frames": r["frames"], "edges_used": r["edges_used"], "edges_dropped": r["edges_dropped"],
                           "pcg_iterations": r["pcg_iterations"], "residual": r["residual"], "state_changes": r["state_changes"],
                           "rot_rms_error_deg": rot_rms_deg(x_ri, g["gt"]), "oracle_rot_rms_error_deg": rot_rms_deg(o["poses"], g["gt"]),
                           "max_abs_R_diff_vs_oracle": float(np.abs(ro.quat_R(x_ri[rows, 3:7]) - o["R"]).max()),
                           "singular_values_of_M_at_that_frame": np.linalg.svd(o["M"][worst], compute_uv=False).tolist(),
                           "frames_with_R_diff_above_1e-8": int((dR > 1e-8).sum()),
                           "oracle_host_s": t_or}
        for start in ("raw", "rot_init"):
            rs = []
            for k in range(args.calls + 1):
                s = handle(grav, **SETTINGS)
                if start == "rot_init":
                    rot_init(s, grav)
                rep = s.solve()
                if k:
                    rs.append(rep)
                x = s.get_poses(g["ids"]); s.close()
            sm = summary(rs)
            dp, dr = synth.pose_errors(x, xr[grav]); gp, gr = synth.pose_errors(x, g["gt"])
            sm.update({"oracle_converged_cost": ref_cost[grav], "cost_rel_diff_vs_oracle": (rs[-1].final_cost - ref_cost[grav]) / ref_cost[grav],
                       "max_pos_err_vs_oracle_m": dp, "max_rot_err_vs_oracle_rad": dr, "max_pos_err_vs_gt_m": gp, "max_rot_err_vs_gt_rad": gr,
                       "rot_rms_error_deg": rot_rms_deg(x, g["gt"])})
            leg["solve_from_" + start] = sm
        out["gravity_rows_and_priors" if grav else "no_gravity"] = leg
    print(json.dumps(out))


if __name__ == "__main__":
    main()
