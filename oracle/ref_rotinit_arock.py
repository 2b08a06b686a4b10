"""ctypes front-end of oracle/_ref/libd2ref_rotinit_arock.so: the REFERENCE's own distributed rotation initialisation
(RotationInitARock<double> in d2pgo/src/rot_init/rotation_initialization_arock.hpp on ARockBase, d2common/src/solver/ARock.cpp)
compiled unmodified by oracle/Makefile.ref against the stand-in headers of oracle/_shim.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_rotinit_arock.py (oracle/pgo_rotinit_arock_oracle.py == reference) and by
tests/golden/make_ref_rotinit_arock_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C

import numpy as np

from oracle.ref import Pin, _p

_PIN = Pin("libd2ref_rotinit_arock.so", "d2pgo")
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


def run(splits, ego, rounds, rho_rot_mat, eta_k, gravity, gravity_sqrt_info=10.0, max_duals=4096):
    """The reference's agents on pgo.arock_split outputs (splits[0] is main_id's), ego [n_a, 7] per split (initial_ego_pose),
    `rounds` synchronous rounds.  Returns one dict per round: per agent (lists in split order) state [n, 3, 3] (rotation states),
    poses [n, 7] (pose states, after the round's delivery), state_changes, and the dual table keys [(neighbour, frame id)],
    yl [K, 9], yr [K, 9] in (neighbour, frame id) order."""
    A = len(splits)
    nf = np.array([len(s["ids"]) for s in splits], np.int32); nl = np.array([len(s["id_a"]) for s in splits], np.int32)
    cat = lambda k, t, w=None: np.ascontiguousarray(np.concatenate([np.asarray(s[k], t).reshape(len(s[k]), -1) if w else np.asarray(s[k], t) for s in splits]))
    ids = cat("ids", np.int64); poses = cat("poses", np.float64, 7); owner = cat("owner", np.int32); fixed = cat("fixed", np.uint8)
    ka = cat("id_a", np.int64); kb = cat("id_b", np.int64); rel = cat("rel", np.float64, 7); S = cat("sqrt_info", np.float64, 36)
    eg = np.ascontiguousarray(np.concatenate([np.asarray(e, np.float64).reshape(-1, 7) for e in ego]))
    self_ids = np.array([s["self_id"] for s in splits], np.int32)
    F = int(nf.sum())
    st = np.zeros((rounds, F, 9)); ps = np.zeros((rounds, F, 7)); chg = np.zeros((rounds, A)); nd = np.zeros((rounds, A), np.int32)
    nb = np.zeros((rounds, A, max_duals), np.int32); fr = np.zeros((rounds, A, max_duals), np.int64)
    yl = np.zeros((rounds, A, max_duals, 9)); yr = np.zeros((rounds, A, max_duals, 9))
    rc = lib().ref_rot_init_arock(C.c_int(A), _p(self_ids), _p(nf), _p(ids), _p(poses), _p(owner), _p(eg), _p(fixed), _p(nl), _p(ka), _p(kb), _p(rel), _p(S),
                                  C.c_double(rho_rot_mat), C.c_double(eta_k), C.c_int(1 if gravity else 0), C.c_double(gravity_sqrt_info), C.c_int(rounds),
                                  _p(st), _p(ps), _p(chg), C.c_int(max_duals), _p(nd), _p(nb), _p(fr), _p(yl), _p(yr))
    assert rc == 0, rc
    off = np.concatenate([[0], np.cumsum(nf)])
    out = []
    for r in range(rounds):
        out.append(dict(state=[st[r, off[a]:off[a + 1]].reshape(-1, 3, 3) for a in range(A)], poses=[ps[r, off[a]:off[a + 1]] for a in range(A)],
                        state_changes=chg[r].copy(),
                        keys=[[(int(n), int(f)) for n, f in zip(nb[r, a, :nd[r, a]], fr[r, a, :nd[r, a]])] for a in range(A)],
                        yl=[yl[r, a, :nd[r, a]] for a in range(A)], yr=[yr[r, a, :nd[r, a]] for a in range(A)]))
    return out
