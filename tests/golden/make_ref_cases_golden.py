"""Freezes what the device-side and g2o tests compare against from the REFERENCE's own code (oracle/_ref/libd2ref.so, built
by oracle/Makefile.ref where the reference sources are present) into tests/golden/ref_cases.npz, so that those tests run
from a plain checkout:
  - reprojection / IMU factor outputs on the seeded windows of tests/test_gpu_vs_reference.py (every observation, in the
    device's tangent layout),
  - RelPoseFactorAD on every 5th edge of the graph of tests/test_pgo.py::test_pgo_edges_on_device_match_the_reference_functor,
  - read_g2o_agent on the files pgo.write_g2o_agents writes for the g2o test graph (with those files' SHA-256),
    and the file write_result_to_g2o writes,
  - PoseLocalParameterization::Plus, its ComputeJacobian and the quaternion average of test_ref_pin's manifold cases.
Run where oracle/_ref/libd2ref.so can be built:  python tests/golden/make_ref_cases_golden.py"""
import hashlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import test_gpu_vs_reference as tgv  # noqa: E402
import test_pgo as tp  # noqa: E402
import test_ref_pin as trp  # noqa: E402
from d2slam_b200 import abi, pgo, synth  # noqa: E402
from oracle import ref  # noqa: E402

BLOCKS = {abi.PROJ_2F1C: [(0, 0), (6, 1), (12, 2)], abi.PROJ_2F2C: [(0, 0), (6, 1), (12, 2), (18, 3)], abi.PROJ_1F2C: [(12, 0), (18, 1)]}


def arrays():
    out = {}
    # reprojection factors: per sampled observation [r (2) | J (2 x 26) in the device's block layout]
    for ci, case in enumerate(tgv.PROJ_CASES):
        pr = synth.make_window(**case)
        pose = {int(i): p for i, p in zip(pr["frame_ids"], pr["poses"])}
        ext = {int(i): p for i, p in zip(pr["cam_ids"], pr["ext"])}
        lam = {int(i): v for i, v in zip(pr["lm_ids"], pr["inv_dep"])}
        td = np.array([pr["td"]])
        want = []
        for o in pr["obs"]:
            t = int(o["type"])
            pi, pj, ea, eb = pose[int(o["frame_a"])], pose.get(int(o["frame_b"])), ext[int(o["cam_a"])], ext.get(int(o["cam_b"]))
            l = np.array([lam[int(o["landmark_id"])]])
            params = {abi.PROJ_2F1C: [pi, pj, ea, l, td], abi.PROJ_2F2C: [pi, pj, ea, eb, l, td], abi.PROJ_1F2C: [ea, eb, l, td]}[t]
            r, Js, _ = ref.proj_eval(t, o["pts_i"], o["pts_j"], o["vel_i"], o["vel_j"], float(o["td_i"]), float(o["td_j"]), 0.0, params)
            w = np.zeros((2, 27)); w[:, 0] = r[:2]
            for off, bi in BLOCKS[t]:
                assert np.all(Js[bi][:, 6] == 0)          # the quaternion's w column of the ambient Jacobian is never written
                w[:, 1 + off:7 + off] = Js[bi][:, :6]
            w[:, 25] = Js[-2][:, 0]; w[:, 26] = Js[-1][:, 0]
            want.append(w)
        out[f"proj{ci}_want"] = np.array(want)

    # IMU factors: r (15), J (15 x 30 tangent), sqrt_info (15 x 15)
    pr = synth.make_window(**tgv.IMU_CASE)
    pose = {int(i): p for i, p in zip(pr["frame_ids"], pr["poses"])}
    sb = {int(i): p for i, p in zip(pr["sb_ids"], pr["sb"])}
    rs, Jrs, sis = [], [], []
    for m in pr["imu"]:
        pre = {f: m[f] for f in ("sum_dt", "delta_p", "delta_q", "delta_v", "jacobian", "covariance")}
        r, Js, si = ref.imu_eval(pre, m["linearized_ba"], m["linearized_bg"], pose[int(m["frame_a"])], sb[int(m["frame_a"])], pose[int(m["frame_b"])], sb[int(m["frame_b"])])
        rs.append(r); Jrs.append(np.concatenate([Js[0][:, :6], Js[1], Js[2][:, :6], Js[3]], axis=1)); sis.append(si)
    out["imu_r"], out["imu_J"], out["imu_sqrt_info"] = np.array(rs), np.array(Jrs), np.array(sis)

    # RelPoseFactorAD on every 5th edge: [r (6) | J_a (6 x 6) | J_b (6 x 6)] in the tangent of the pose manifold
    g, S = tp.relpose_graph()
    idx, want = [], []
    for e in range(0, len(g["ea"]), 5):
        a, b = g["ea"][e], g["eb"][e]
        r, Ja, Jb = ref.relpose_ad_eval(g["init"][a], g["init"][b], g["rel"][e], S[e])
        idx.append(e); want.append(np.concatenate([r, (Ja @ trp.plus_jacobian(g["init"][a])).ravel(), (Jb @ trp.plus_jacobian(g["init"][b])).ravel()]))
    out["relpose_idx"] = np.array(idx, np.int32); out["relpose_want"] = np.array(want)

    # g2o: the reference's reader on the files written here, and the file the reference's writer produces
    with tempfile.TemporaryDirectory() as td:
        g, S = tp.g2o_agents_graph()
        agents = pgo.write_g2o_agents(td, g["ids"], g["init"], g["id_a"], g["id_b"], g["rel"], S.reshape(-1, 36))
        for a in agents:
            path = os.path.join(td, f"{a}.g2o")
            out[f"g2o_agent{a}_sha256"] = np.array(hashlib.sha256(open(path, "rb").read()).hexdigest())
            for k, v in ref.g2o_read(path, max_agent_id=len(agents) - 1).items():
                out[f"g2o_agent{a}_{k}"] = v
            r0 = ref.g2o_read(path, max_agent_id=0)
            out[f"g2o_agent{a}_n_filtered"] = np.array([len(r0["v_id"]), len(r0["e_id_a"])])
        g, info = tp.g2o_written_graph()
        path = os.path.join(td, "out.g2o")
        ref.g2o_write(path, g["ids"], g["init"], g["id_a"], g["id_b"], g["rel"], info)
        out["g2o_written"] = np.frombuffer(open(path, "rb").read(), np.uint8)

    # manifold helpers
    xs, ds, qs = trp.manifold_cases()
    out["pose_plus"] = np.array([ref.pose_plus(x, d) for x, d in zip(xs, ds)])
    out["pose_plus_jacobian"] = ref.pose_plus_jacobian(xs[0])
    out["average_quat"] = ref.average_quats(qs)
    return out


def main():
    out = arrays()
    np.savez_compressed(os.path.join(HERE, "ref_cases.npz"), **out)
    print("wrote", len(out), "arrays,", os.path.getsize(os.path.join(HERE, "ref_cases.npz")), "bytes")


if __name__ == "__main__":
    main()
