"""Distributed rotation-initialisation benchmark (d2pgo's RotationInitARock before the ARock solve, pgo_mode 1): the bench's
pose graph as 8 agents on one GPU.

Workload: pgo.make_pose_graph(seed=7) (8 trajectories x 1250 poses, 40 000 edges) split into 8 agents by pgo.arock_split, as
tools/pgo_arock_bench.py does; agent 0's head frame fixed.  Two parameter sets, both with d2pgo_test_multi.launch's rho_rot_mat
0.16 and eta_k 0.9: gravity rows off, and on (ego poses from pgo.make_gravity_case).  For each, pgo.arock_rot_init_run up to
--max-rounds rounds with rotInitial's gate (state_changes < 1e-2 after more than 10 solves) and reports:
  - device ms per round (sum over the agents that stepped of d2pgo_rot_init_report.device_ms), mean and max;
  - the round at which each agent passed the gate (None: not within --max-rounds);
  - the RMS rotation error to ground truth of the frames at their owners, before, after the distributed initialisation, and
    after the centralised d2pgo_rot_init on the whole graph with the same gravity rows;
  - --arock-rounds following d2pgo_arock_step rounds (pgo.arock_run; bench.py pgo_leg's LM settings, ARock defaults with
    eta_k 0.9), with and without the rotation-initialisation phase: the whole graph's cost at the agents' own poses over the
    centralised optimum, and the largest distance between two agents' copies of a frame, after the first and the last round.
Prints one JSON line with the card name and power limit read in the same run.  Writes nothing.

    python tools/pgo_rotinit_arock_bench.py [--max-rounds 100] [--arock-rounds 20]
"""
import argparse
import json
import os
import sys

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(_v, "1")
import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from d2slam_b200 import pgo  # noqa: E402
from pgo_4dof_bench import SETTINGS, card  # noqa: E402
from pgo_arock_bench import OPTIMUM, disagreement, own_poses, whole_cost  # noqa: E402

ROT = dict(rho_rot_mat=0.16)   # d2pgo_test_multi.launch:13-16 (with eta_k 0.9, the ARock config of the agents)
AROCK = dict(eta_k=0.9)


def rot_rms(x, gt):
    """RMS over frames of the rotation angle between attitudes x and gt [N, 7] (rad)"""
    d = np.abs(np.sum(np.asarray(x)[:, 3:7] / np.linalg.norm(np.asarray(x)[:, 3:7], axis=1, keepdims=True) * gt[:, 3:7], axis=1)).clip(0, 1)
    return float(np.sqrt(np.mean((2 * np.arccos(d)) ** 2)))


def agents_of(splits, ego):
    return [pgo.ArockAgent(sp, ego_poses=None if ego is None else ego[sp["pos"]], solver_kw=SETTINGS, **AROCK) for sp in splits]


def arock_phase(g, agents, rounds, c_opt):
    hist = []

    def after(k, ags, reps):
        x = own_poses(g, ags, lambda a: a.poses())
        hist.append({"round": k + 1, "own_pose_cost_over_optimum": whole_cost(6, g, x) / c_opt,
                     "max_copy_distance_m": disagreement(6, [(a.split["ids"], a.poses()) for a in ags]),
                     "device_ms": float(sum(q.device_ms for q in reps))})
    pgo.arock_run(agents, rounds, after)
    return {"first": hist[0], "last": hist[-1]} if hist else {}


def leg(g, splits, ego, max_rounds, arock_rounds, c_opt):
    grav = ego is not None
    # the centralised rotation initialisation of the whole graph, same rows
    s = pgo.PgoSolver()
    s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    rep_c = s.rot_init(g["ids"] if grav else None, ego, enable_gravity_prior=int(grav))
    x_c = s.get_poses(g["ids"]); s.close()
    # the distributed one
    agents = agents_of(splits, ego)
    per_round = []
    done = pgo.arock_rot_init_run(agents, max_rounds, after_round=lambda k, ags, reps: per_round.append(
        sum(r["device_ms"] for r in reps if r is not None)), enable_gravity_prior=int(grav), **ROT)
    x_d = own_poses(g, agents, lambda a: a.poses())
    with_init = arock_phase(g, agents, arock_rounds, c_opt)
    for a in agents:
        a.close()
    fresh = agents_of(splits, ego)
    without = arock_phase(g, fresh, arock_rounds, c_opt)
    for a in fresh:
        a.close()
    ms = np.array(per_round)
    return {"gravity_rows": grav, "rounds_run": len(per_round), "converged_round_per_agent": done,
            "device_ms_per_round": {"mean": float(ms.mean()), "max": float(ms.max())},
            "rotation_rms_to_ground_truth_rad": {"initial_guess": rot_rms(g["init"], g["gt"]), "distributed": rot_rms(x_d, g["gt"]),
                                                 "centralised_d2pgo_rot_init": rot_rms(x_c, g["gt"])},
            "centralised_device_ms": rep_c["device_ms"],
            "arock_after_rot_init": with_init, "arock_without_rot_init": without}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-rounds", type=int, default=100)
    ap.add_argument("--arock-rounds", type=int, default=20)
    args = ap.parse_args()
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)   # + 7 connecting closures = 40 000 edges
    ego = pgo.make_gravity_case(g, seed=7)["ego"]
    pos = {int(i): k for k, i in enumerate(g["ids"])}
    splits = [dict(pgo.arock_split(g, a)) for a in range(8)]
    for sp in splits:
        sp["pos"] = np.array([pos[int(i)] for i in sp["ids"]])
    s = pgo.PgoSolver(**OPTIMUM)
    s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    c_opt = s.solve().final_cost; s.close()
    out = {"metric": "pgo_rotinit_arock", "card": card(),
           "settings": {"rot_init": ROT, "arock": AROCK, "local_lm": SETTINGS, "gate": {"eps": 1e-2, "min_rounds": 10}},
           "workload": f"{len(g['ids'])} poses / {len(g['id_a'])} edges as 8 ARock agents (one per trajectory) on one GPU, synchronous schedule",
           "whole_graph_optimum_cost": c_opt,
           "gravity_off": leg(g, splits, None, args.max_rounds, args.arock_rounds, c_opt),
           "gravity_on": leg(g, splits, ego, args.max_rounds, args.arock_rounds, c_opt)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
