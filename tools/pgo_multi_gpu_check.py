"""torchrun worker: the pose graph's edges sharded over the ranks (e % world), J^T J p all-reduced over NCCL inside
libd2ba (include/d2pgo.h) -- every rank must end on the single-rank solution (rank 0 also solves the whole graph alone).
--dof 4 runs the same check on the graph's 4-DoF version (pgo.pose_graph_to_4d, RelPoseFactor4D).  --gravity adds a gravity
prior on every pose (pgo.make_gravity_case, full S), the priors split over the ranks like the edges (k % world)."""
import argparse
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from d2slam_b200 import pgo, synth  # noqa: E402
from d2slam_b200.solver import comm_unique_id  # noqa: E402


def pose_errors(x, y, dof):
    if dof == 6:
        return synth.pose_errors(x, y)
    return np.linalg.norm(x[:, :3] - y[:, :3], axis=1).max(), np.abs(pgo.normalize_angle(x[:, 3] - y[:, 3])).max()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dof", type=int, choices=(6, 4), default=6)
    ap.add_argument("--gravity", action="store_true", help="6-DoF with a gravity prior on every pose")
    args = ap.parse_args()
    dof = args.dof
    if args.gravity and dof != 6:
        ap.error("--gravity needs --dof 6")
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); lr = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    g = pgo.make_pose_graph(seed=11, n_agents=4, poses_per_agent=80, loops=400)
    if dof == 4:
        g = pgo.pose_graph_to_4d(g, seed=11)
    if args.gravity:
        ego = pgo.make_gravity_case(g, seed=11)["ego"]
        gS = pgo.GRAVITY_SQRT_INFO * np.eye(3) + 2.0 * np.random.default_rng(11).normal(size=(len(g["ids"]), 3, 3))
    kw = dict(device=lr, max_iterations=25, pcg_max_iterations=800, pcg_tolerance=1e-10, lambda0=0.0, function_tolerance=1e-13, pose_dof=dof)

    def load(s, sel, gsel=None):
        if args.gravity:
            s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"][sel], g["id_b"][sel], g["rel"][sel], g["sqrt_info"][sel])
            s.add_gravity_priors(g["ids"][gsel], ego[gsel], gS[gsel])
        elif dof == 4:
            s.set_poses_4d(g["ids"], g["init"], g["fixed"]); s.add_edges_4d(g["id_a"][sel], g["id_b"][sel], g["rel"][sel], g["sqrt_info"][sel])
        else:
            s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"][sel], g["id_b"][sel], g["rel"][sel], g["sqrt_info"][sel])

    def poses(s):
        return s.get_poses_4d(g["ids"]) if dof == 4 else s.get_poses(g["ids"])
    sel = np.arange(rank, len(g["id_a"]), world)
    s = pgo.PgoSolver(**kw)
    load(s, sel, np.arange(rank, len(g["ids"]), world))
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid.copy_(torch.tensor(list(comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(uid, 0)
    s.comm_init(bytes(uid.cpu().tolist()), rank, world)
    rep = s.solve()
    x = poses(s)
    # all ranks hold the same poses, bit for bit
    t = torch.tensor(x, device="cuda"); t0 = t.clone(); dist.broadcast(t0, 0)
    same = bool((t == t0).all().item())
    ok = same and rep.final_cost < rep.initial_cost
    if rank == 0:
        s1 = pgo.PgoSolver(**kw)
        load(s1, np.arange(len(g["id_a"])), np.arange(len(g["ids"])))
        r1 = s1.solve()
        dp, dr = pose_errors(x, poses(s1), dof)
        print(f"pgo multi ({dof}-DoF{' + gravity priors' if args.gravity else ''}): cost {rep.final_cost:.9e} vs single {r1.final_cost:.9e}; pose diff {dp:.3e} m {dr:.3e} rad; lm its {rep.iterations}/{r1.iterations}; ranks identical {same}")
        ok = ok and abs(rep.final_cost - r1.final_cost) <= 1e-9 * r1.final_cost and dp <= 1e-6 and dr <= 1e-6
    flag = torch.tensor([1 if ok else 0], device="cuda"); dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("PGO_MULTI_GPU_CHECK " + ("PASS" if flag.item() else "FAIL"))
    dist.destroy_process_group()
    sys.exit(0 if flag.item() else 1)


if __name__ == "__main__":
    main()
