"""ctypes front-end of oracle/_ref/libd2ref.so: the REFERENCE's own factor classes (compiled unmodified from
/root/reference by oracle/Makefile.ref against the stand-in headers of oracle/_shim), and `Pin`, which builds and loads
every library of oracle/Makefile.ref for its front-end module.

TEST INFRASTRUCTURE ONLY: used by tests/test_ref_pin.py (oracle restatement == reference, and the golden vectors under
tests/golden/ref_factors.npz) and by tests/golden/make_ref_golden.py.  Nothing under d2slam_b200/ imports it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("D2SLAM_REF", "/root/reference")


class Pin:
    """One reference pin library, oracle/_ref/<name>, built from the sources under REF_ROOT/<subtree>.  Where the reference
    tree is absent (the GPU machines) the prebuilt file is used as is.  `setup(lib)` runs once on the freshly loaded library."""

    def __init__(self, name, subtree, setup=None):
        self.name, self.subtree, self.setup, self._lib = name, subtree, setup, None

    def so_path(self):
        return os.path.join(_HERE, "_ref", self.name)

    def _buildable(self):
        return os.path.isdir(os.path.join(REF_ROOT, self.subtree))

    def available(self):
        return os.path.exists(self.so_path()) or self._buildable()

    def build(self, force=False):
        """Compile the library where its reference sources lie (a no-op when it is up to date) and return its path."""
        so = self.so_path()
        if self._buildable():
            subprocess.check_call(["make", "-C", _HERE, "-f", "Makefile.ref", "-s", f"REF={REF_ROOT}", f"_ref/{self.name}"] + (["-B"] if force else []))
        if not os.path.exists(so):
            raise RuntimeError(f"oracle/_ref/{self.name} missing and the reference tree is not present to build it")
        return so

    def lib(self):
        if self._lib is None:
            self._lib = C.CDLL(self.build())
            if self.setup is not None:
                self.setup(self._lib)
        return self._lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def configure(focal_length=460.0, depth_sqrt_inf=20.0, g_norm=9.805, acc_n=0.1, gyr_n=0.05, acc_w=0.002, gyr_w=0.0004):
    lib().ref_configure(*[C.c_double(v) for v in (focal_length, depth_sqrt_inf, g_norm, acc_n, gyr_n, acc_w, gyr_w)])


_PIN = Pin("libd2ref.so", "d2vins", setup=lambda _: configure())
so_path, available, build, lib = _PIN.so_path, _PIN.available, _PIN.build, _PIN.lib


_BLOCKS = {0: (7, 7, 7, 1, 1), 1: (7, 7, 7, 7, 1, 1), 2: (7, 7, 1, 1), 3: (7, 7, 7, 1, 1)}


def proj_eval(typ, pts_i, pts_j, vel_i, vel_j, td_i, td_j, depth_j, params):
    """params: list of arrays in the factor's own block order.  -> (r, [J_k (rows x size_k)], tangent_base (2x3))."""
    sizes = _BLOCKS[int(typ)]
    rows = 3 if int(typ) == 3 else 2
    ps = [np.ascontiguousarray(np.atleast_1d(p), dtype=np.float64) for p in params]
    assert [len(p) for p in ps] == list(sizes), ([len(p) for p in ps], sizes)
    parr = (C.c_void_p * len(ps))(*[_p(p) for p in ps])
    r = np.zeros(rows)
    Js = [np.zeros((rows, s)) for s in sizes]
    jarr = (C.c_void_p * len(Js))(*[_p(j) for j in Js])
    tb = np.zeros(6)
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (pts_i, pts_j, vel_i, vel_j)]
    n = lib().ref_proj_eval(C.c_int(int(typ)), _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), C.c_double(td_i), C.c_double(td_j), C.c_double(depth_j),
                            parr, _p(r), jarr, _p(tb))
    assert n == rows, n
    return r, Js, tb.reshape(2, 3)


def preintegrate(dt, acc, gyr, ba, bg):
    dt = np.ascontiguousarray(dt, dtype=np.float64); acc = np.ascontiguousarray(acc, dtype=np.float64); gyr = np.ascontiguousarray(gyr, dtype=np.float64)
    ba = np.ascontiguousarray(ba, dtype=np.float64); bg = np.ascontiguousarray(bg, dtype=np.float64)
    out = np.zeros(11 + 450)
    lib().ref_preintegrate(C.c_int(len(dt)), _p(dt), _p(acc), _p(gyr), _p(ba), _p(bg), _p(out))
    return {"sum_dt": out[0], "delta_p": out[1:4].copy(), "delta_q": out[4:8].copy(), "delta_v": out[8:11].copy(),
            "jacobian": out[11:236].copy(), "covariance": out[236:461].copy()}


def imu_eval(pre, lin_ba, lin_bg, pose_i, sb_i, pose_j, sb_j):
    ps = [np.ascontiguousarray(p, dtype=np.float64) for p in (pose_i, sb_i, pose_j, sb_j)]
    parr = (C.c_void_p * 4)(*[_p(p) for p in ps])
    r = np.zeros(15); Js = [np.zeros((15, s)) for s in (7, 9, 7, 9)]
    jarr = (C.c_void_p * 4)(*[_p(j) for j in Js])
    si = np.zeros(225)
    f = [np.ascontiguousarray(pre[k], dtype=np.float64).ravel() for k in ("delta_p", "delta_q", "delta_v")]
    ba = np.ascontiguousarray(lin_ba, dtype=np.float64); bg = np.ascontiguousarray(lin_bg, dtype=np.float64)
    jac = np.ascontiguousarray(pre["jacobian"], dtype=np.float64).ravel(); cov = np.ascontiguousarray(pre["covariance"], dtype=np.float64).ravel()
    n = lib().ref_imu_eval(C.c_double(float(pre["sum_dt"])), _p(f[0]), _p(f[1]), _p(f[2]), _p(ba), _p(bg), _p(jac), _p(cov), parr, _p(r), jarr, _p(si))
    assert n == 15, n
    return r, Js, si.reshape(15, 15)


def consensus_eval(t_ref, q_ref, t_tilde, theta_tilde, rho_T, rho_theta, pose):
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (t_ref, q_ref, t_tilde, theta_tilde, pose)]
    r = np.zeros(6); J = np.zeros((6, 7))
    n = lib().ref_consensus_eval(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), C.c_double(rho_T), C.c_double(rho_theta), _p(a[4]), _p(r), _p(J))
    assert n == 6, n
    return r, J


def relpose_ad_eval(pose_a, pose_b, rel7, sqrt_info):
    """RelPoseFactorAD (RelPoseFactor.hpp:68-135): residual (6) and the ambient Jacobians (6 x 7 each) by dual numbers."""
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (pose_a, pose_b, rel7, np.asarray(sqrt_info).reshape(36))]
    r = np.zeros(6); Ja = np.zeros((6, 7)); Jb = np.zeros((6, 7))
    n = lib().ref_relpose_ad_eval(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(r), _p(Ja), _p(Jb))
    assert n == 6, n
    return r, Ja, Jb


def loss_correct(r, J, huber_a):
    """ResidualInfo::Evaluate's loss section (BaseParamResInfo.cpp:71-92) on a given residual / Jacobian."""
    r = np.ascontiguousarray(r, dtype=np.float64); J = np.ascontiguousarray(J, dtype=np.float64)
    ro = np.zeros_like(r); Jo = np.zeros_like(J)
    n = lib().ref_loss_correct(C.c_int(J.shape[0]), C.c_int(J.shape[1]), _p(r), _p(J), C.c_double(huber_a), _p(ro), _p(Jo))
    assert n == len(r), n
    return ro, Jo


def admm_replay(present, traj, relaxation_alpha, rho_T, rho_theta):
    """The reference's ConsensusSolver::solve loop (ConsensusSolver.cpp:39-235) replaying a prescribed trajectory of local
    poses: present [A][B] (agent a holds block b), traj [K+1][A][B][7] -> z [K][A][B][7], tilde [K][A][B][6] and the residuals
    [K][A][B][6] of the ConsenusPoseFactor objects it created at every step (evaluated at the step's local poses)."""
    present = np.ascontiguousarray(present, dtype=np.uint8); traj = np.ascontiguousarray(traj, dtype=np.float64)
    K = traj.shape[0] - 1; A, B = present.shape
    z = np.zeros((K, A, B, 7)); tl = np.zeros((K, A, B, 6)); rs = np.zeros((K, A, B, 6))
    rc = lib().ref_admm_replay(C.c_int(A), C.c_int(B), C.c_int(K), C.c_double(relaxation_alpha), C.c_double(rho_T), C.c_double(rho_theta),
                               _p(present), _p(traj), _p(z), _p(tl), _p(rs))
    assert rc == 0, rc
    return z, tl, rs


PRIOR_SIZE = (7, 7, 9, 1, 1); PRIOR_EFF = (6, 6, 9, 1, 1)   # POSE, EXTRINSIC, SPEED_BIAS, TD, LANDMARK


def prior_eval(kinds, x0, x, A, b):
    """PriorFactor(keep_params, A, b).Evaluate(x) (prior_factor.cpp:45-90, toJacRes :132-177): residual (m) and the m x m
    tangent Jacobian assembled from the per-block Jacobians' leftCols(eff_size) (the remaining columns are asserted zero)."""
    kinds = np.ascontiguousarray(kinds, dtype=np.int32); x0 = np.ascontiguousarray(x0, dtype=np.float64); x = np.ascontiguousarray(x, dtype=np.float64)
    A = np.ascontiguousarray(A, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64); m = len(b)
    r = np.zeros(m); J = np.zeros(sum(m * PRIOR_SIZE[k] for k in kinds))
    n = lib().ref_prior_eval(C.c_int(len(kinds)), _p(kinds), _p(x0), _p(x), C.c_int(m), _p(A), _p(b), _p(r), _p(J))
    assert n == m, n
    Jt = np.zeros((m, m)); off = eo = 0
    for k in kinds:
        blk = J[off:off + m * PRIOR_SIZE[k]].reshape(m, PRIOR_SIZE[k])
        assert np.all(blk[:, PRIOR_EFF[k]:] == 0.0)
        Jt[:, eo:eo + PRIOR_EFF[k]] = blk[:, :PRIOR_EFF[k]]; off += m * PRIOR_SIZE[k]; eo += PRIOR_EFF[k]
    return r, Jt


def marginalize(pr, remove_frame_ids, huber_delta=1.0, max_m=512):
    """The reference's Marginalizer::marginalize over the reference factor objects of one synthetic window `pr` (a
    d2slam_b200.synth.Problem): -> kept block refs, their linearisation points, and the new prior as (J, e0)."""
    from d2slam_b200 import abi
    obs = np.ascontiguousarray(pr["obs"]); imu = np.ascontiguousarray(pr["imu"])
    lm_ids = np.ascontiguousarray(pr["lm_ids"], dtype=np.int64)
    base = {}
    for o in obs:
        base.setdefault(int(o["landmark_id"]), int(o["frame_a"]))
    lm_base = np.array([base[int(i)] for i in lm_ids], dtype=np.int64)
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    i64 = lambda a: np.ascontiguousarray(a, dtype=np.int64)
    if pr.get("prior") is not None:
        A, b, refs, x0 = pr["prior"]; A = f64(A); b = f64(b); refs = np.ascontiguousarray(refs, dtype=abi.blockref_dtype); x0 = f64(x0); m = len(b)
    else:
        A = b = x0 = np.zeros(1); refs = np.zeros(1, dtype=abi.blockref_dtype); m = 0
    rem = i64(remove_frame_ids)
    nblk = C.c_int(); mo = C.c_int(); refs_out = np.zeros(256, dtype=abi.blockref_dtype); x0_out = np.zeros(256 * 9); J = np.zeros(max_m * max_m); e0 = np.zeros(max_m)
    fid = i64(pr["frame_ids"]); cid = i64(pr["cam_ids"])
    rc = lib().ref_marginalize(C.c_int(len(fid)), _p(fid), _p(f64(pr["poses"])), _p(f64(pr["sb"])), C.c_int(len(cid)), _p(cid), _p(f64(pr["ext"])), C.c_double(float(pr["td"])),
                               C.c_int(len(lm_ids)), _p(lm_ids), _p(f64(pr["inv_dep"])), _p(lm_base), C.c_int(len(obs)), _p(obs), C.c_int(len(imu)), _p(imu),
                               C.c_int(m), _p(A), _p(b), C.c_int(len(refs) if m else 0), _p(refs), _p(x0), C.c_int(len(rem)), _p(rem), C.c_double(huber_delta),
                               C.byref(nblk), _p(refs_out), _p(x0_out), C.byref(mo), _p(J), _p(e0), C.c_int(max_m))
    assert rc == 0, rc
    mm = mo.value; refs_out = refs_out[: nblk.value].copy()
    nx = int(sum(abi.KIND_SIZE[int(k)] for k in refs_out["kind"]))
    return refs_out, x0_out[:nx].copy(), J[: mm * mm].reshape(mm, mm).copy(), e0[:mm].copy()


def g2o_read(path, max_agent_id=100000, cap=200000):
    """read_g2o_agent (d2pgo/test/posegraph_g2o.cpp:133-175) on one file -> vertices (agent, keyframe id, pose7), edges
    (agent_a, id_a, agent_b, id_b, rel7, information 6x6)."""
    nv = C.c_int(); ne = C.c_int()
    va = np.zeros(cap, np.int32); vi = np.zeros(cap, np.int64); vp = np.zeros((cap, 7))
    ea = np.zeros(cap, np.int32); eia = np.zeros(cap, np.int64); eb = np.zeros(cap, np.int32); eib = np.zeros(cap, np.int64); er = np.zeros((cap, 7)); ei = np.zeros((cap, 36))
    rc = lib().ref_g2o_read(path.encode(), C.c_int(max_agent_id), C.c_int(cap), C.c_int(cap), C.byref(nv), _p(va), _p(vi), _p(vp), C.byref(ne), _p(ea), _p(eia), _p(eb), _p(eib), _p(er), _p(ei))
    assert rc == 0, rc
    n, m = nv.value, ne.value
    return dict(v_agent=va[:n], v_id=vi[:n], v_pose=vp[:n], e_agent_a=ea[:m], e_id_a=eia[:m], e_agent_b=eb[:m], e_id_b=eib[:m], e_rel=er[:m], e_info=ei[:m].reshape(m, 6, 6))


def g2o_write(path, v_id, v_pose, e_id_a, e_id_b, e_rel, e_info):
    """write_result_to_g2o (posegraph_g2o.cpp:197-232)."""
    a = [np.ascontiguousarray(v_id, np.int64), np.ascontiguousarray(v_pose, np.float64), np.ascontiguousarray(e_id_a, np.int64), np.ascontiguousarray(e_id_b, np.int64),
         np.ascontiguousarray(e_rel, np.float64), np.ascontiguousarray(np.asarray(e_info).reshape(-1, 36), np.float64)]
    rc = lib().ref_g2o_write(path.encode(), C.c_int(len(a[0])), _p(a[0]), _p(a[1]), C.c_int(len(a[2])), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]))
    assert rc == 0, rc


def relpose4d_eval(pose_a4, pose_b4, rel7, sqrt_info4):
    """RelPoseFactor4D (RelPoseFactor.hpp:196-238): poses [x y z yaw]; residual (4) and the 4 x 4 Jacobians by dual numbers."""
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (pose_a4, pose_b4, rel7, np.asarray(sqrt_info4).reshape(16))]
    r = np.zeros(4); Ja = np.zeros((4, 4)); Jb = np.zeros((4, 4))
    n = lib().ref_relpose4d_eval(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(r), _p(Ja), _p(Jb))
    assert n == 4, n
    return r, Ja, Jb


def pose_plus(x, delta):
    x = np.ascontiguousarray(x, dtype=np.float64); d = np.ascontiguousarray(delta, dtype=np.float64); o = np.zeros(7)
    lib().ref_pose_plus(_p(x), _p(d), _p(o))
    return o


def pose_plus_jacobian(x):
    x = np.ascontiguousarray(x, dtype=np.float64); J = np.zeros((7, 6))
    lib().ref_pose_plus_jacobian(_p(x), _p(J))
    return J


def qleft_qright(q):
    q = np.ascontiguousarray(q, dtype=np.float64); L = np.zeros((4, 4)); R = np.zeros((4, 4))
    lib().ref_qleft_qright(_p(q), _p(L), _p(R))
    return L, R


def average_quats(qs):
    qs = np.ascontiguousarray(qs, dtype=np.float64); o = np.zeros(4)
    lib().ref_average_quats(C.c_int(len(qs)), _p(qs), _p(o))
    return o
