"""ctypes front-end of oracle/_ref/libd2ref_pcm.so: d2pgo's PCM loop outlier rejection as the REFERENCE's own code
(SwarmLocalOutlierRejection, FMC maxCliqueHeu), compiled unmodified from the reference tree by oracle/Makefile.ref against the
stand-in headers of oracle/_shim.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_pcm.py (oracle/pcm_oracle.py == reference) and by
tests/golden/make_ref_pcm_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C

import numpy as np

from oracle.ref import Pin, _p

_PIN = Pin("libd2ref_pcm.so", "d2pgo")
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


def pcm(case, is_4dof, thres=1.635, pos_cov=4e-3, yaw_cov=4e-5, rel_key="rel"):
    """SwarmLocalOutlierRejection::OutlierRejectionLoopEdges (swarm_outlier_rejection.cpp:46-303) fed every loop of `case`
    (the d2slam_b200.pgo.make_pcm_case layout) once -> (good mask, smd of every tested pair in the reference's call order:
    groups by (max drone id, min drone id) ascending, rows i ascending, j ascending)."""
    fid = np.ascontiguousarray(case["frame_ids"], np.int64); fag = np.ascontiguousarray(case["frame_agent"], np.int32)
    ego = np.ascontiguousarray(case["ego"], np.float64); ka = np.ascontiguousarray(case["kf_a"], np.int64); kb = np.ascontiguousarray(case["kf_b"], np.int64)
    rel = np.ascontiguousarray(case[rel_key], np.float64); si = np.ascontiguousarray(np.asarray(case["sqrt_info"]).reshape(-1, 36), np.float64)
    n = len(ka); cap = max(n * (n - 1) // 2, 1)
    good = np.zeros(max(n, 1), np.uint8); smd = np.zeros(cap); ns = C.c_int64()
    rc = lib().ref_pcm(C.c_int(int(is_4dof)), C.c_double(thres), C.c_double(pos_cov), C.c_double(yaw_cov), C.c_int(len(fid)), _p(fid), _p(fag), _p(ego),
                       C.c_int(n), _p(ka), _p(kb), _p(rel), _p(si), _p(good), _p(smd), C.c_int64(cap), C.byref(ns))
    assert rc >= 0, rc
    return good[:n].astype(bool), smd[: ns.value].copy()


def fmc_heu(adj):
    """FMC::maxCliqueHeu (findCliqueHeu.cpp:124-243) on a symmetric boolean adjacency -> the clique as FMC lists it."""
    adj = np.asarray(adj, bool); n = len(adj)
    ptr = np.zeros(n + 1, np.int32); ptr[1:] = np.cumsum(adj.sum(1))
    nb = np.ascontiguousarray(np.nonzero(adj)[1], np.int32)
    out = np.zeros(max(n, 1), np.int32)
    k = lib().ref_fmc_heu(C.c_int(n), _p(ptr), _p(nb if len(nb) else np.zeros(1, np.int32)), _p(out))
    return out[:k].tolist()
