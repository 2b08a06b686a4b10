"""ARock distributed pose-graph benchmark (d2pgo's pgo_mode 1): the bench's pose graph as 8 agents on one GPU.

Workload: pgo.make_pose_graph(seed=7) (8 trajectories x 1250 poses, 40 000 edges); agent s = trajectory s with its sub-graph
from pgo.arock_split (its own odometry and every loop between frames it knows); agent 0's head frame fixed.  Both
configurations (4-DoF through pgo.pose_graph_to_4d, and 6-DoF perturbation duals), the node's parameters (d435_multi.yaml:
rho_frame_T 0.7, rho_frame_theta 0.625, eta_k 0.1), each local solve with bench.py pgo_leg's LM settings, the synchronous
broadcast schedule (pgo.arock_run).  Per round: the device ms of all agents' steps (sum of their d2pgo_report.device_ms),
the largest distance between two agents' copies of a frame, and the whole graph's cost at the agents' own poses (each frame
from its owner) against the cost d2pgo_solve reaches on the whole graph.  The CPU reference is the oracle's ARock round
(oracle/pgo_arock_oracle.py, sparse-direct local solves, one host thread) for the first --oracle-rounds rounds.  Prints one
JSON line with the card name and power limit read in the same run.  Writes nothing.

    python tools/pgo_arock_bench.py [--rounds 20] [--oracle-rounds 1]
"""
import argparse
import json
import os
import sys
import time

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(_v, "1")
import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo  # noqa: E402
from pgo_4dof_bench import SETTINGS, card  # noqa: E402

NODE = dict(rho_frame_T=0.7, rho_frame_theta=0.625, eta_k=0.1)   # config/realsense_d435/d435_multi.yaml
OPTIMUM = dict(max_iterations=200, pcg_max_iterations=500, pcg_tolerance=1e-6, lambda0=1e-4, function_tolerance=1e-12)


def whole_cost(dof, gg, x):
    from oracle import pgo4d_oracle as p4
    from oracle import pgo_oracle as po
    if dof == 4:
        return p4.cost_4d(x, gg["ea"], gg["eb"], gg["rel"], gg["sqrt_info"])
    r = po.edges_eval(np.asarray(x), np.asarray(gg["ea"]), np.asarray(gg["eb"]), np.asarray(gg["rel"]), np.asarray(gg["sqrt_info"]).reshape(-1, 6, 6))[0]
    return 0.5 * float(np.sum(r * r))


def own_poses(gg, agents, get):
    """every frame's pose as its owner agent holds it"""
    pos = {int(i): k for k, i in enumerate(gg["ids"])}
    x = np.array(gg["init"], np.float64)
    for a in agents:
        xs = get(a)
        for i, f in enumerate(a.split["ids"] if hasattr(a, "split") else a.ids):
            if int(f) // 1_000_000 == a.self_id:
                x[pos[int(f)]] = xs[i]
    return x


def disagreement(dof, agents_x):
    seen = {}
    for ids, x in agents_x:
        for f, p in zip(ids, x):
            seen.setdefault(int(f), []).append(p)
    worst = 0.0
    for ps in seen.values():
        for p in ps[1:]:
            worst = max(worst, float(np.linalg.norm(p[:3] - ps[0][:3])))
    return worst


def leg(dof, gg, rounds, oracle_rounds):
    n_agents = int(np.max(gg["agent"])) + 1
    # the whole graph on one handle: the optimum the agents' own poses are measured against
    s = pgo.PgoSolver(pose_dof=dof, **OPTIMUM)
    if dof == 4:
        s.set_poses_4d(gg["ids"], gg["init"], gg["fixed"]); s.add_edges_4d(gg["id_a"], gg["id_b"], gg["rel"], gg["sqrt_info"])
    else:
        s.set_poses(gg["ids"], gg["init"], gg["fixed"]); s.add_edges(gg["id_a"], gg["id_b"], gg["rel"], gg["sqrt_info"])
    r = s.solve(); c_opt = r.final_cost; s.close()
    splits = [pgo.arock_split(gg, a) for a in range(n_agents)]
    agents = [pgo.ArockAgent(sp, solver_kw=SETTINGS, **NODE) for sp in splits]
    per_round = []

    def after(k, ags, reps):
        x = own_poses(gg, ags, lambda a: a.poses())
        per_round.append({"round": k + 1, "device_ms": float(sum(q.device_ms for q in reps)), "lm_iterations": int(sum(q.iterations for q in reps)),
                          "max_copy_distance_m": disagreement(dof, [(a.split["ids"], a.poses()) for a in ags]),
                          "own_pose_cost_over_optimum": whole_cost(dof, gg, x) / c_opt})
    t0 = time.perf_counter()
    pgo.arock_run(agents, rounds, after)
    wall = time.perf_counter() - t0
    duals = [sum(len(a.s.arock_duals(int(n))[0]) for n in a.s.arock_neighbours()) for a in agents]
    for a in agents:
        a.close()
    out = {"agents": n_agents, "frames_per_agent": [len(sp["ids"]) for sp in splits], "edges_per_agent": [len(sp["id_a"]) for sp in splits],
           "duals_per_agent": duals, "whole_graph_optimum_cost": c_opt, "initial_cost_over_optimum": whole_cost(dof, gg, gg["init"]) / c_opt,
           "rounds": per_round, "host_wall_s_all_rounds": wall}
    if oracle_rounds:
        from oracle import pgo_arock_oracle as ao
        orc = [ao.OracleAgent(sp, **NODE) for sp in splits]
        t0 = time.perf_counter()
        ao.arock_run(orc, oracle_rounds)
        out["cpu_oracle"] = {"what": "numpy + scipy sparse-direct local solves to convergence (oracle/pgo_arock_oracle.py), 1 host thread",
                             "rounds": oracle_rounds, "s_per_round": (time.perf_counter() - t0) / oracle_rounds}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--oracle-rounds", type=int, default=1, help="oracle rounds timed on the CPU (0 = none)")
    args = ap.parse_args()
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)   # + 7 connecting closures = 40 000 edges
    h = pgo.pose_graph_to_4d(g, seed=7)
    out = {"metric": "pgo_arock", "card": card(), "settings": {"local_lm": SETTINGS, "arock": NODE, "whole_graph": OPTIMUM},
           "workload": f"{len(g['ids'])} poses / {len(g['id_a'])} edges as 8 ARock agents (one per trajectory) on one GPU, synchronous broadcast schedule",
           "dof4": leg(4, h, args.rounds, args.oracle_rounds), "dof6": leg(6, g, args.rounds, args.oracle_rounds)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
