"""ctypes front-end of oracle/_ref/libd2ref_rotinit.so: the REFERENCE's own chordal rotation initialisation
(RotationInitialization<double>::solve in d2pgo/src/rot_init/rotation_initialization_base.hpp, with pgostate.hpp and
utils.hpp) included unmodified from the reference tree by oracle/Makefile.ref against the stand-in headers of oracle/_shim.

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_rotinit.py (oracle/pgo_rotinit_oracle.py == reference) and by
tests/golden/make_ref_rotinit_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C

import numpy as np

from oracle.ref import Pin, _p

_PIN = Pin("libd2ref_rotinit.so", "d2pgo")
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


def rot_init(ids, poses, fixed, id_a, id_b, rel, sqrt_info, gravity=False, gravity_sqrt_info=10.0, ego_ids=None, ego_poses=None):
    """The reference's RotationInitialization<double> (enable_float32 off) on frames ids / poses / fixed flags with their ego
    poses (identity where none is given) and loops (id_a, id_b, rel7, sqrt_info36): setFixedFrameId per fixed frame, solve().
    Returns dict(frames = the solved free frame ids ascending, M [F, 3, 3] = their rotation states after the call, R [F, 3, 3] =
    the rotations of their new attitudes, poses [n, 7] = every pose state after the call, state_changes, dropped = loops that
    gave no rows)."""
    ids = np.ascontiguousarray(ids, np.int64); n = len(ids)
    poses = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(n, 7)); fx = np.ascontiguousarray(fixed, np.uint8)
    ego = np.tile(np.array([0, 0, 0, 0, 0, 0, 1.0]), (n, 1))
    if ego_ids is not None:
        where = {int(i): k for k, i in enumerate(ids)}
        for i, p in zip(np.asarray(ego_ids, np.int64), np.asarray(ego_poses, np.float64).reshape(-1, 7)):
            if int(i) in where:
                ego[where[int(i)]] = p
    ego = np.ascontiguousarray(ego)
    ka = np.ascontiguousarray(id_a, np.int64); kb = np.ascontiguousarray(id_b, np.int64); E = len(ka)
    rel = np.ascontiguousarray(np.asarray(rel, np.float64).reshape(E, 7)); S = np.ascontiguousarray(np.asarray(sqrt_info, np.float64).reshape(E, 36))
    rot = np.zeros((n, 9)); out = np.zeros((n, 7)); solved = np.zeros(n, np.uint8); chg = C.c_double(); dropped = C.c_int32()
    rc = lib().ref_rot_init(C.c_int(n), _p(ids), _p(poses), _p(fx), _p(ego), C.c_int(E), _p(ka), _p(kb), _p(rel), _p(S), C.c_int(1 if gravity else 0),
                            C.c_double(gravity_sqrt_info), _p(rot), _p(out), _p(solved), C.byref(chg), C.byref(dropped))
    assert rc == 0, rc
    sel = solved.astype(bool)
    from oracle.pgo_rotinit_oracle import quat_R
    return dict(frames=ids[sel], M=rot[sel].reshape(-1, 3, 3), R=quat_R(out[sel, 3:7]), poses=out, state_changes=np.float64(chg.value),
                dropped=np.int64(dropped.value))
