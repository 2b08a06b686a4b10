"""ctypes front-end of oracle/_ref/libd2ref_gravity.so: the REFERENCE's own perturbation-mode PGO functors
(GravityPriorPerturbAD, RelPoseFactorPerturbAD) included unmodified from the reference tree by oracle/Makefile.gravity against
the stand-in headers of oracle/_shim, evaluated with doubles (residual) and dual numbers (Jacobians).

TEST INFRASTRUCTURE ONLY: used by tests/test_pgo_gravity.py (oracle/pgo_gravity_oracle.py == reference) and by
tests/golden/make_ref_gravity_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.ref import REF_ROOT

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def so_path():
    return os.path.join(_HERE, "_ref", "libd2ref_gravity.so")


def available():
    return os.path.exists(so_path()) or os.path.isdir(os.path.join(REF_ROOT, "d2common"))


def build(force=False):
    """Compile the reference's functors where they lie (only possible where the reference tree exists)."""
    so = so_path()
    if os.path.isdir(os.path.join(REF_ROOT, "d2common")):
        subprocess.check_call(["make", "-C", _HERE, "-f", "Makefile.gravity", "-s", f"REF={REF_ROOT}"] + (["-B"] if force else []))
    if not os.path.exists(so):
        raise RuntimeError("oracle/_ref/libd2ref_gravity.so missing and the reference tree is not present to build it")
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a, n):
    a = np.ascontiguousarray(np.asarray(a, np.float64).ravel())
    assert a.size == n, (a.size, n)
    return a


def gravity_prior_eval(ego7, S, q0, pose6):
    """GravityPriorPerturbAD(ego_pose, S, q0) (GravityPrior.hpp:8-46) at the perturbation block [p, theta]:
    r (3) and J (3 x 6, by dual numbers)."""
    a = [_f64(ego7, 7), _f64(S, 9), _f64(q0, 4), _f64(pose6, 6)]
    r = np.zeros(3); J = np.zeros((3, 6))
    n = lib().ref_gravity_prior_eval(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(r), _p(J))
    assert n == 3, n
    return r, J


def relpose_perturb_eval(rel7, S, qa0, qb0, a6, b6):
    """RelPoseFactorPerturbAD(rel, S, qa0, qb0) (RelPoseFactor.hpp:138-195) at the perturbation blocks [p_a, theta_a],
    [p_b, theta_b]: r (6) and J_a, J_b (6 x 6, by dual numbers)."""
    a = [_f64(rel7, 7), _f64(S, 36), _f64(qa0, 4), _f64(qb0, 4), _f64(a6, 6), _f64(b6, 6)]
    r = np.zeros(6); Ja = np.zeros((6, 6)); Jb = np.zeros((6, 6))
    n = lib().ref_relpose_perturb_eval(*[_p(x) for x in a], _p(r), _p(Ja), _p(Jb))
    assert n == 6, n
    return r, Ja, Jb
