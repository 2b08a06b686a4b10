"""ctypes front-end of oracle/_ref/libd2ref_pcm_stream.so: d2pgo's PCM as the REFERENCE's own code kept across calls
(SwarmLocalOutlierRejection) and FMC::maxCliqueHeuIncremental, compiled unmodified from the reference tree by
oracle/Makefile.ref_pcm_stream against the stand-in headers of oracle/_shim.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_pcm_stream.py (oracle/pcm_stream_oracle.py == reference) and by
tests/golden/make_ref_pcm_stream_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.ref import REF_ROOT, Pin, _p


class _StreamPin(Pin):
    """A Pin built by oracle/Makefile.ref_pcm_stream (which includes Makefile.ref)."""

    def build(self, force=False):
        so = self.so_path()
        if self._buildable():
            here = os.path.dirname(os.path.abspath(__file__))
            subprocess.check_call(["make", "-C", here, "-f", "Makefile.ref_pcm_stream", "-s", f"REF={REF_ROOT}", f"_ref/{self.name}"] + (["-B"] if force else []))
        if not os.path.exists(so):
            raise RuntimeError(f"oracle/_ref/{self.name} missing and the reference tree is not present to build it")
        return so


def _setup(L):
    L.ref_pcm_stream_new.restype = C.c_void_p
    L.ref_pcm_stream_free.argtypes = [C.c_void_p]


_PIN = _StreamPin("libd2ref_pcm_stream.so", "d2pgo", _setup)
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


class PcmStream:
    """One SwarmLocalOutlierRejection kept across calls (redundant = true, incremental_pcm = false), fed as D2PGO feeds it:
    call(frames new since the last call, loops = every loop so far) -> (good mask over the loops given, smd of the pairs the
    call tested in the reference's order: groups by (max drone id, min drone id) ascending, new rows in arrival order, j
    ascending)."""

    def __init__(self, is_4dof, thres=1.635, pos_cov=4e-3, yaw_cov=4e-5):
        self._h = C.c_void_p(lib().ref_pcm_stream_new(C.c_int(int(is_4dof)), C.c_double(thres), C.c_double(pos_cov), C.c_double(yaw_cov)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ref_pcm_stream_free(self._h); self._h = None

    def call(self, frame_ids, frame_agent, ego, loop_ids, kf_a, kf_b, rel7, sqrt_info36):
        fid = np.ascontiguousarray(frame_ids, np.int64); fag = np.ascontiguousarray(frame_agent, np.int32)
        eg = np.ascontiguousarray(np.asarray(ego, np.float64).reshape(-1, 7)); lid = np.ascontiguousarray(loop_ids, np.int64)
        ka = np.ascontiguousarray(kf_a, np.int64); kb = np.ascontiguousarray(kf_b, np.int64)
        rel = np.ascontiguousarray(np.asarray(rel7, np.float64).reshape(-1, 7)); si = np.ascontiguousarray(np.asarray(sqrt_info36, np.float64).reshape(-1, 36))
        n = len(lid); cap = max(n * (n - 1) // 2, 1)
        good = np.zeros(max(n, 1), np.uint8); smd = np.zeros(cap); ns = C.c_int64()
        rc = lib().ref_pcm_stream_call(self._h, C.c_int(len(fid)), _p(fid), _p(fag), _p(eg), C.c_int(n), _p(lid), _p(ka), _p(kb), _p(rel), _p(si), _p(good),
                                       _p(smd), C.c_int64(cap), C.byref(ns))
        assert rc >= 0, rc
        return good[:n].astype(bool), smd[: ns.value].copy()


def fmc_heu_inc(adj, num_new, prev):
    """FMC::maxCliqueHeuIncremental (findCliqueHeuInc.cpp:11-99) on a symmetric boolean adjacency whose last num_new vertices
    are new, under the bound prev -> its return value."""
    adj = np.asarray(adj, bool); n = len(adj)
    ptr = np.zeros(n + 1, np.int32); ptr[1:] = np.cumsum(adj.sum(1))
    nb = np.ascontiguousarray(np.nonzero(adj)[1], np.int32)
    return int(lib().ref_fmc_heu_inc(C.c_int(n), _p(ptr), _p(nb if len(nb) else np.zeros(1, np.int32)), C.c_int(num_new), C.c_int(prev)))
