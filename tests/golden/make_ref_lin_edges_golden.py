"""Freezes the REFERENCE's per-observation values (oracle/_ref/libd2ref.so: the projection factor classes' Evaluate and
ResidualInfo's loss section) on the edge observations of tests/test_ba_lin_variants.py's catalogue -- outliers, far / near /
negative inverse depths, bearings on and just off the optical axis and behind the camera, negated quaternions -- at each
configuration those windows run with, into tests/golden/ref_lin_edges.npz: per observation the factor type, (s_px, s_d,
delta), the loss-corrected residual (3) and Jacobian (3 x 30, [pose_i 7 | pose_j 7 | ext_a 7 | ext_b 7 | lambda | td]).
Run where oracle/_ref/libd2ref.so can be built:  python tests/golden/make_ref_lin_edges_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import test_ba_lin_variants as tlv  # noqa: E402
from oracle import ref  # noqa: E402


def arrays():
    typ, cfg, rs, Js = [], [], [], []
    try:
        for name, cfg_name, k in tlv.edge_cases():
            t, o, x, cfgv = tlv.case_inputs(name, cfg_name, k)
            r, J, _ = tlv.ref_obs_eval(t, o, *x, *cfgv)
            typ.append(t); cfg.append(cfgv); rs.append(r); Js.append(J)
    finally:
        ref.configure()
    return {"typ": np.array(typ, np.int32), "cfg": np.array(cfg, np.float64), "r": np.array(rs), "J": np.array(Js)}


def main():
    np.savez_compressed(os.path.join(HERE, "ref_lin_edges.npz"), **arrays())


if __name__ == "__main__":
    main()
