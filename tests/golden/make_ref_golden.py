"""Freezes outputs of the REFERENCE's own factor classes (oracle/_ref/libd2ref.so, built from /root/reference by
oracle/Makefile.ref) on the seeded cases of tests/test_ref_pin.py into tests/golden/ref_factors.npz.
Run in the build container (the GPU box has no /root/reference):  python tests/golden/make_ref_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import test_ref_pin as t  # noqa: E402
from oracle import ref  # noqa: E402


def arrays():
    out = {}
    for i, c in enumerate(t.proj_cases()):
        r, Js, tb = ref.proj_eval(c["typ"], c["pts_i"], c["pts_j"], c["vel_i"], c["vel_j"], c["td_i"], c["td_j"], c["depth"], t.ref_params(c))
        out[f"proj{i}_r"] = r; out[f"proj{i}_tb"] = tb
        for k, J in enumerate(Js):
            out[f"proj{i}_J{k}"] = J
    for i, c in enumerate(t.imu_cases()):
        pre = ref.preintegrate(c["dt"], c["acc"], c["gyr"], c["ba0"], c["bg0"])
        r, Js, si = ref.imu_eval(pre, c["ba0"], c["bg0"], c["pi"], c["sbi"], c["pj"], c["sbj"])
        out[f"imu{i}_pre_jacobian"] = pre["jacobian"]; out[f"imu{i}_pre_covariance"] = pre["covariance"]
        out[f"imu{i}_sqrt_info"] = si; out[f"imu{i}_r"] = r
        for k, J in enumerate(Js):
            out[f"imu{i}_J{k}"] = J
    for i, c in enumerate(t.cons_cases()):
        r, J = ref.consensus_eval(c["z"][:3], c["z"][3:7], c["tt"], c["th"], c["rho_T"], c["rho_theta"], c["x"])
        out[f"cons{i}_r"] = r; out[f"cons{i}_J"] = J
    for i, c in enumerate(t.relpose_cases()):
        r, Ja, Jb = ref.relpose_ad_eval(c["pa"], c["pb"], c["rel"], c["S"])
        out[f"relpose{i}_r"] = r; out[f"relpose{i}_Ja"] = Ja; out[f"relpose{i}_Jb"] = Jb
    for i, c in enumerate(t.loss_cases()):
        r, J = ref.loss_correct(c["r"], c["J"], c["a"])
        out[f"loss{i}_r"] = r; out[f"loss{i}_J"] = J
    for i, c in enumerate(t.prior_cases()):
        out[f"prior{i}_r"], out[f"prior{i}_J"] = ref.prior_eval(c["kinds"], c["x0"], c["x"], c["A"], c["b"])
    for i, c in enumerate(t.relpose4d_cases()):
        out[f"relpose4d{i}_r"], out[f"relpose4d{i}_Ja"], out[f"relpose4d{i}_Jb"] = ref.relpose4d_eval(c["pa"], c["pb"], c["rel"], c["S"])
    ref.configure()
    for i, kw in enumerate(t.MARG_CASES):
        pr = t.synth.make_window(**kw)
        out[f"marg{i}_refs"], out[f"marg{i}_x0"], out[f"marg{i}_J"], out[f"marg{i}_e0"] = ref.marginalize(pr, [int(pr["frame_ids"][0])])
    _, present, traj = t.admm_trajectory()
    out["admm_z"], out["admm_tilde"], out["admm_res"] = ref.admm_replay(present, traj, t.ADMM_KW["relaxation_alpha"], t.ADMM_KW["rho_frame_T"], t.ADMM_KW["rho_frame_theta"])
    return out


def main():
    out = arrays()
    np.savez_compressed(os.path.join(HERE, "ref_factors.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
