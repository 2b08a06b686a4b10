"""ctypes binding of oracle/_ref/libd2ref_arock.so: the reference's own ARock loop (d2common/src/solver/ARock.cpp compiled
unmodified by oracle/Makefile.ref against the stand-in headers of oracle/_shim, ARockPGO's message handling restated in
oracle/ref_arock_driver.cpp) replaying given local solutions.
TEST INFRASTRUCTURE: imported by tests/ only."""
import ctypes as C

import numpy as np

from oracle.ref import Pin


def _setup(lib):
    lib.ref_arock_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


_PIN = Pin("libd2ref_arock.so", "d2common", setup=_setup)
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


def run(self_ids, frames, owners, init, solved, rho_T, rho_theta, eta, init_zero=False, max_n=256):
    """The reference's ARock loop over len(self_ids) agents, synchronous schedule.  frames / owners / init: per agent, its frame
    ids, their owners and their initial states [n, D] in dual coordinates; solved[r][a]: agent a's local solution of round r
    [n, D].  Returns per round a list over the agents of dict(keys [(neighbour, frame)], yl [K, D], yr [K, D], fac [K, D + D^2])
    -- the dual table after the step and r | J of the step's proximal factors at the solution, (neighbour, frame) ascending."""
    A = len(self_ids); D = np.asarray(init[0]).shape[1]; R = len(solved)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    sid = np.ascontiguousarray(self_ids, np.int32); nf = np.array([len(f) for f in frames], np.int32)
    fid = np.ascontiguousarray(np.concatenate(frames), np.int64); own = np.ascontiguousarray(np.concatenate(owners), np.int32)
    x0 = np.ascontiguousarray(np.concatenate(init), np.float64)
    xs = np.ascontiguousarray(np.stack([np.concatenate(s) for s in solved]), np.float64)
    n = np.zeros(R * A, np.int32); keys = np.zeros((R * A, max_n, 2), np.int64)
    yl = np.zeros((R * A, max_n, D)); yr = np.zeros((R * A, max_n, D)); fac = np.zeros((R * A, max_n, D + D * D))
    rc = lib().ref_arock_run(A, D, R, p(sid), rho_T, rho_theta, eta, int(init_zero), p(nf), p(fid), p(own), p(x0), p(xs), max_n,
                              p(n), p(keys), p(yl), p(yr), p(fac))
    assert rc == 0 and n.max(initial=0) <= max_n
    out = []
    for r in range(R):
        row = []
        for a in range(A):
            s, k = r * A + a, n[r * A + a]
            row.append(dict(keys=[(int(u), int(v)) for u, v in keys[s, :k]], yl=yl[s, :k], yr=yr[s, :k], fac=fac[s, :k]))
        out.append(row)
    return out
