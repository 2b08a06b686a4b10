"""BA reprojection linearisation, entry by entry, in every kernel variant d2ba_finalize routes observations to.

d2ba_finalize sends each group (a run of observations that share their parameter blocks) to one of eight kernels; the
launcher (launch_proj_lin, d2ba_kernels.cu) maps the job index to the instantiation:

    0 k_proj_lin<2,2>   1 k_proj_lin<4,2>   2 k_proj_lin<2,4>   3 k_proj_lin<4,4>              (NCT, KR)
    4 k_proj_lin_pp<true,false>   5 <false,false>   6 <true,true>   7 <false,true>            (SHIFT0, REC12)

``predict_routing`` restates that rule from the problem alone and D2BA_DBG_LIN_JOBS must equal it.  The catalogue below is
a set of small windows that together reach every variant, with the edges where reprojection kernels go wrong applied to
windows of both kernel families: residuals on both sides of the Huber delta, gross outliers, far / near / negative inverse
depths, bearings on the optical axis, just off it and behind the camera, negated quaternions, and non-default
focal_length, depth_sqrt_inf and huber_delta (including the loss switched off).

Each entry of Hcc, gc, Hll, gl, W and the cost the device forms is compared with a long-double sum of the CPU oracle's
loss-corrected per-observation terms at the device's own state, within

    |dH_ab| <= 2 (C_J + m_ab) eps sum_{k,q} Jb_kqa Jb_kqb

where Jb is each per-observation entry floored at the inf-norm of its own segment of that row (translation, rotation),
lambda, td and the residual at the magnitude of the terms they are differences of (``proj_floors``), and m_ab counts the
terms.  C_J is four times the largest disagreement
between the oracle and the reference's own factor classes over the catalogue, in units of eps Jb (the needs_ref test
measures it; tests/golden/ref_lin_edges.npz freezes the reference values of the edge observations for plain checkouts).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

from d2slam_b200 import abi, synth

EPS = np.finfo(np.float64).eps
LD = np.longdouble
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_lin_edges.npz")
N_SM = 132                # H100 SXM; the GPU tests read the device's own count
# 4 x the largest oracle / reference disagreement over the catalogue, in units of eps Jb (test_oracle_matches_reference_classes
# measures 85 211: the depth row's rotation entries of a landmark at lambda = 1e-4, which cancel to 1e-4 of their terms)
C_J = 3.5e5
HUBER_DEFAULT = 1.0


# ---------------------------------------------------------------------------------------------------------- routing
def _blocks(pr):
    pose = {int(f): i for i, f in enumerate(pr["frame_ids"])}
    ext = {int(c): i for i, c in enumerate(pr["cam_ids"])}
    lm = {int(l): i for i, l in enumerate(pr["lm_ids"])}
    out = []
    for o in pr["obs"]:
        t = int(o["type"])
        pi = pj = ea = eb = -1
        if t != abi.PROJ_DEPTH_PRIOR:
            ea = ext[int(o["cam_a"])]
            if t in (abi.PROJ_2F2C, abi.PROJ_1F2C):
                eb = ext[int(o["cam_b"])]
            if t != abi.PROJ_1F2C:
                pi, pj = pose[int(o["frame_a"])], pose[int(o["frame_b"])]
        out.append((t, pi, pj, ea, eb, lm[int(o["landmark_id"])]))
    return out


def predict_tpj(problems, n_sm=N_SM):
    """Tiles per job of a handle (d2ba_finalize): the estimated tile count over 8 jobs per SM, clamped to [1, 8]."""
    tiles_est = sum(len(p["obs"]) for p in problems) // 32 + len(problems)
    return max(1, min(8, tiles_est // (n_sm * 8)))


def predict_routing(pr, tpj_target=1):
    """The D2BA_DBG_LIN_JOBS view of one window restated from the problem: d2ba_finalize's group rule (slots, need_ext,
    need_td, nct, rows, shift0, the fast-path test), the balanced split of a group's tiles into jobs, the 96-byte record
    rule that moves the fast-path jobs to the REC12 instantiations, and motion_needed."""
    from test_ba_solve_shapes import predict_plan
    obs = _blocks(pr)
    pc, ec = np.asarray(pr["pose_const"]).astype(bool), np.asarray(pr["ext_const"]).astype(bool)
    td_free = not pr["td_const"]
    stamps = [v for o in pr["obs"] if int(o["type"]) != abi.PROJ_DEPTH_PRIOR for v in (float(o["td_i"]), float(o["td_j"]))]
    same_stamp = bool(stamps) and min(stamps) == max(stamps) == float(pr["td"])
    groups = {}
    for o in obs:
        groups.setdefault(o[:5], []).append(o)
    out = {v: dict.fromkeys(abi.LIN_JOBS_FIELDS, 0) for v in abi.LIN_VARIANTS}
    for key in sorted(groups):
        t, pi, pj, ea, eb = key
        cols = [pi >= 0 and not pc[pi], pj >= 0 and not pc[pj], ea >= 0 and not ec[ea], eb >= 0 and not ec[eb]]
        if t == abi.PROJ_DEPTH_PRIOR:
            cols = [False] * 4
        src = [s for s in range(4) if cols[s]]
        need_td = td_free and t != abi.PROJ_DEPTH_PRIOR
        need_ext = any(s >= 2 for s in src)
        nct = 2 if (len(src) <= 2 and not need_td) else 4
        rows = 3 if t == abi.PROJ_2F1C_DEPTH else (1 if t == abi.PROJ_DEPTH_PRIOR else 2)
        v = (1 if nct == 4 else 0) + (2 if rows == 3 else 0)
        shift0 = not need_td and t != abi.PROJ_DEPTH_PRIOR and same_stamp
        if v == 0 and not need_ext and t in (abi.PROJ_2F1C, abi.PROJ_2F2C) and src == [0, 1]:
            v = 4 if shift0 else 5
        cnt = len(groups[key]); ntile = (cnt + 31) // 32; njob = (ntile + tpj_target - 1) // tpj_target
        c = out[abi.LIN_VARIANTS[v]]
        c["groups"] += 1; c["jobs"] += njob; c["tiles"] += ntile; c["obs"] += cnt
        for j in range(njob):
            c["max_tiles_per_job"] = max(c["max_tiles_per_job"], ntile * (j + 1) // njob - ntile * j // njob)
    if predict_plan(pr)["rec_stride"] == 12:
        V = abi.LIN_VARIANTS
        out[V[6]], out[V[4]] = out[V[4]], out[V[6]]
        out[V[7]], out[V[5]] = out[V[5]], out[V[7]]
    out["motion_needed"] = int(bool(stamps) and (td_free or not same_stamp))
    out["tpj_target"] = tpj_target
    return out


# ---------------------------------------------------------------------------------------------------------- catalogue
def _vision(pr, anchor_const=False):
    """Vision only: no IMU factor, no speed-bias block, no prior; pose 0 constant only when asked (a free anchor pose is
    what the fast path needs).  The state starts 1 mm / 0.06 deg / 1 % from the truth, so that the residual norms spread
    around the default Huber delta (1.5 px of bearing noise)."""
    pr["imu"] = pr["imu"][:0]; pr["sb_ids"] = pr["sb_ids"][:0]; pr["sb"] = pr["sb"][:0]
    pr["prior"] = None; pr["consensus"] = None
    rng = np.random.default_rng(len(pr["obs"]))
    pr["poses"] = synth.pose_plus(pr["poses_gt"], np.concatenate([rng.normal(0, 1e-3, (len(pr["poses_gt"]), 3)),
                                                                   rng.normal(0, 1e-3, (len(pr["poses_gt"]), 3))], axis=1))
    pr["inv_dep"] = pr["inv_dep_gt"] * (1 + 0.01 * rng.normal(size=len(pr["inv_dep_gt"])))
    pc = np.zeros(len(pr["frame_ids"]), np.uint8)
    pc[0] = 1 if anchor_const else 0
    pr["pose_const"] = pc
    return pr


def _reanchor(pr, every=3):
    """Move the anchor of every `every`-th landmark from frame 0 to frame 1 (mono tracks): its observation from frame 1
    becomes the anchor bearing, and frame 0 becomes an observing frame."""
    f0, f1 = pr["frame_ids"][0], pr["frame_ids"][1]
    o = pr["obs"]
    out = []
    for li, l in enumerate(pr["lm_ids"]):
        rec = o[o["landmark_id"] == l]
        if li % every or not np.any(rec["frame_b"] == f1):
            out.append(rec); continue
        a = rec[rec["frame_b"] == f1][0]
        new = rec[rec["frame_b"] != f1].copy()
        back = a.copy()
        back["frame_b"] = f0; back["pts_j"] = a["pts_i"]; back["vel_j"] = a["vel_i"]; back["td_j"] = a["td_i"]
        new = np.concatenate([back[None], new])
        new["frame_a"] = f1; new["pts_i"] = a["pts_j"]; new["vel_i"] = a["vel_j"]; new["td_i"] = a["td_j"]
        out.append(new)
    pr["obs"] = np.concatenate(out)
    return pr


def _depth(pr):
    ids, tptr, tobs = pr["tracks"]
    tobs = tobs.copy(); tobs["depth_mea"] = 1
    pr["obs"] = synth.tracks_to_obs(ids, tptr, tobs, fuse_dep=True, min_d=0.3, max_d=50.0)
    return pr


EDGE_FAMILIES = ("outlier", "lambda_far", "lambda_near", "lambda_negative", "on_axis", "off_axis", "behind", "negated_quat")


def _edges(pr, seed):
    """Every edge family on one window; pr["edges"][family] lists the observation indices it touches."""
    rng = np.random.default_rng(seed)
    o = pr["obs"].copy()
    lm_index = {int(l): i for i, l in enumerate(pr["lm_ids"])}
    reproj = np.nonzero(o["type"] != abi.PROJ_DEPTH_PRIOR)[0]
    pick = rng.permutation(reproj)
    n_out = max(1, len(reproj) // 10)
    edges = {}
    out_idx = pick[:n_out]
    d = rng.normal(size=(n_out, 3)); d[:, 2] = np.abs(d[:, 2]) + 0.3
    o["pts_j"][out_idx] = d / np.linalg.norm(d, axis=1, keepdims=True)
    edges["outlier"] = out_idx
    rest = pick[n_out:]
    o["pts_j"][rest[0]] = (0.0, 0.0, 1.0)
    o["pts_j"][rest[1]] = np.array([1e-9, -1e-9, 1.0]) / np.linalg.norm([1e-9, -1e-9, 1.0])
    o["pts_j"][rest[2]] = np.array([0.1, 0.2, -1.0]) / np.linalg.norm([0.1, 0.2, -1.0])
    o["pts_i"][rest[3]] = np.array([-0.1, 0.05, -1.0]) / np.linalg.norm([-0.1, 0.05, -1.0])
    edges["on_axis"], edges["off_axis"], edges["behind"] = rest[:1], rest[1:2], rest[2:4]
    pr["obs"] = o
    lam = pr["inv_dep"].copy()
    lms = [int(x) for x in o["landmark_id"][rest[4:7]]]
    for fam, l, v in zip(("lambda_far", "lambda_near", "lambda_negative"), lms, (1e-4, 10.0, -0.2)):
        lam[lm_index[l]] = v
        edges[fam] = np.nonzero(o["landmark_id"] == l)[0]
    pr["inv_dep"] = lam
    poses = pr["poses"].copy()
    neg = [1, 3]
    poses[neg, 3:7] *= -1
    pr["poses"] = poses
    ext = pr["ext"].copy(); ext[-1, 3:7] *= -1; pr["ext"] = ext
    fa = set(int(f) for f in pr["frame_ids"][neg])
    edges["negated_quat"] = np.nonzero([int(x["frame_a"]) in fa or int(x["frame_b"]) in fa for x in o])[0][:8]
    pr["edges"] = edges
    return pr


def _remote(seed):
    pr = synth.make_swarm(seed=seed, n_agents=2, n_frames=15, only_agents=[0], shared_per_pair=10, n_landmarks=60)[0]
    pr["consensus"] = None; pr["prior"] = None
    return pr


CATALOGUE = {
    # fast path, 96-byte records: td constant and equal to every stamp / differing from them (the td shift applies)
    "mono_s0": lambda: _vision(synth.make_window(seed=301, n_frames=6, n_landmarks=60)),
    "mono_shift": lambda: _vision(synth.make_window(seed=302, n_frames=6, n_landmarks=60, td_offset=0.002)),
    # constant frame 0, every landmark anchored in frame 1: k_proj_lin<2,2> with one slot (frame 0 observing), fast path
    # at stride 16 (100 landmarks: 4-tile groups)
    "anchor_s0": lambda: _reanchor(_vision(synth.make_window(seed=303, n_frames=5, n_landmarks=100), anchor_const=True), 1),
    "anchor_shift": lambda: _reanchor(_vision(synth.make_window(seed=304, n_frames=5, n_landmarks=100, td_offset=0.002), anchor_const=True), 1),
    # stereo, second extrinsic free, td constant: <2,2> with need_ext (1F2C), <4,2>, fast path at stride 32
    "stereo_ext": lambda: _vision(synth.make_window(seed=305, n_frames=5, n_landmarks=50, cams="stereo", estimate_extrinsic=True)),
    # stereo, td free: <4,2>
    "stereo_td": lambda: _vision(synth.make_window(seed=306, n_frames=5, n_landmarks=50, cams="stereo", estimate_td=True, td_offset=0.002)),
    # depth tracks: <2,4> and the depth prior (<2,2> without slots); with td free: <4,4>
    "depth": lambda: _depth(_vision(synth.make_window(seed=307, n_frames=5, n_landmarks=60))),
    "depth_td": lambda: _depth(_vision(synth.make_window(seed=308, n_frames=5, n_landmarks=60, estimate_td=True, td_offset=0.002))),
    # quad cameras: 1F2C groups with no column at all
    "quad": lambda: _vision(synth.make_window(seed=309, n_frames=4, n_landmarks=80, cams="quad")),
    # two agents: the remote frames form a leaf, so the fast path writes 128-byte records (IMU factors kept: they make
    # the own frames the hub)
    "a2": lambda: _remote(310),
    # the edge families on fast-path windows and on generic windows
    "mono_s0_edges": lambda: _edges(_vision(synth.make_window(seed=311, n_frames=6, n_landmarks=60)), 1),
    "anchor_shift_edges": lambda: _edges(_reanchor(_vision(synth.make_window(seed=312, n_frames=5, n_landmarks=90, td_offset=0.002), anchor_const=True), 2), 2),
    "stereo_td_edges": lambda: _edges(_vision(synth.make_window(seed=313, n_frames=5, n_landmarks=50, cams="stereo", estimate_td=True, td_offset=0.002)), 3),
    "depth_edges": lambda: _edges(_depth(_vision(synth.make_window(seed=314, n_frames=5, n_landmarks=60))), 4),
}
# windows in a handle of their own with a non-default configuration (one fast-path and one generic window each);
# "huber_at" puts delta on one observation's residual norm (1e-12 relative)
CONFIGS = {
    "focal": dict(focal_length=300.0, depth_sqrt_inf=5.0, huber_delta=0.5),
    "huber_off": dict(huber_delta=-1.0),
    "huber_at": None,
}
CONFIG_WINDOWS = ("mono_s0_edges", "depth_edges")

_CACHE = {}


def problem(name):
    if name not in _CACHE:
        _CACHE[name] = CATALOGUE[name]()
    return _CACHE[name]


def config_of(cfg_name, win_name):
    """Solver keyword arguments of a configuration variant for one window."""
    if cfg_name == "huber_at":
        pr = problem(win_name)
        norms = [np.sqrt(np.sum(t["r"][:t["rows"]] ** 2)) for t in _raw_terms(pr, state_of_problem(pr), {})]
        k = int(np.argsort(norms)[len(norms) // 2])
        return dict(huber_delta=float(norms[k]) * (1 + 1e-12))
    return dict(CONFIGS[cfg_name]) if cfg_name else {}


def bench(shift):
    return _vision(synth.make_window(seed=4242, n_frames=11, n_landmarks=300, td_offset=0.002 if shift else 0.0))


def load(pr, solver, window=None):
    args = () if window is None else (window,)
    solver.set_blocks(*args, abi.POSE, pr["frame_ids"], pr["poses"], pr["pose_const"])
    solver.set_blocks(*args, abi.EXTRINSIC, pr["cam_ids"], pr["ext"], pr["ext_const"])
    if len(pr["sb_ids"]):
        solver.set_blocks(*args, abi.SPEED_BIAS, pr["sb_ids"], pr["sb"], None)
    solver.set_blocks(*args, abi.TD, np.zeros(1, np.int64), np.array([pr["td"]]), np.array([pr["td_const"]], np.uint8))
    solver.set_blocks(*args, abi.LANDMARK, pr["lm_ids"], pr["inv_dep"], None)
    solver.add_proj(*args, pr["obs"])
    if len(pr["imu"]):
        solver.add_imu(*args, pr["imu"])


# ---------------------------------------------------------------------------------------------------------- oracle terms
def state_of_problem(pr):
    return dict(pose=pr["poses"].copy(), ext=pr["ext"].copy(), sb=pr["sb"].copy(), lm=pr["inv_dep"].copy(), td=float(pr["td"]))


def state_of_device(s, w, pr):
    st = dict(pose=s.get_blocks(w, abi.POSE, pr["frame_ids"]), ext=s.get_blocks(w, abi.EXTRINSIC, pr["cam_ids"]),
              lm=s.get_blocks(w, abi.LANDMARK, pr["lm_ids"])[:, 0], td=float(s.get_blocks(w, abi.TD, np.zeros(1, np.int64))[0, 0]))
    st["sb"] = s.get_blocks(w, abi.SPEED_BIAS, pr["sb_ids"]) if len(pr["sb_ids"]) else np.zeros((0, 9))
    return st


def _obs_const(o):
    from oracle import orc
    c = orc.OrcObsConst()
    c.pts_i[:] = o["pts_i"]; c.pts_j[:] = o["pts_j"]; c.vel_i[:] = o["vel_i"]; c.vel_j[:] = o["vel_j"]
    c.td_i = float(o["td_i"]); c.td_j = float(o["td_j"])
    c.inv_depth_j = 1.0 / float(o["depth"]) if float(o["depth"]) != 0 else 0.0
    tb = np.zeros(6)
    orc.lib().orc_tangent_base(abi.ptr(np.ascontiguousarray(o["pts_j"], dtype=np.float64)), abi.ptr(tb))
    c.tangent_base[:] = tb
    return c


def orc_obs_eval(typ, o, pose_i, pose_j, ext_a, ext_b, lam, td, s_px, s_d):
    """The oracle's per-observation evaluation (orc_proj_eval / orc_depth_prior_eval) before the loss: r (3), J (3 x 30)
    in the layout [pose_i 7 | pose_j 7 | ext_a 7 | ext_b 7 | lambda | td] (ambient pose columns, the 7th is zero)."""
    from oracle import orc
    L = orc.lib()
    r = np.zeros(3); J = np.zeros((3, 30))
    if typ == abi.PROJ_DEPTH_PRIOR:
        jl = np.zeros(1)
        L.orc_depth_prior_eval(C.c_double(lam), C.c_double(float(o["depth"])), C.c_double(s_d), abi.ptr(r), abi.ptr(jl))
        J[0, 28] = jl[0]
        return r, J, 1
    rows = 3 if typ == abi.PROJ_2F1C_DEPTH else 2
    blk = [np.zeros(rows * 7) for _ in range(4)]
    Jl = np.zeros(3); Jt = np.zeros(3)
    z7 = np.zeros(7); z7[6] = 1.0
    f = lambda a: np.ascontiguousarray(a if a is not None else z7, dtype=np.float64)   # noqa: E731
    c = _obs_const(o)
    L.orc_proj_eval(C.c_int(typ), C.byref(c), C.c_double(s_px), C.c_double(s_d), abi.ptr(f(pose_i)), abi.ptr(f(pose_j)),
                    abi.ptr(f(ext_a)), abi.ptr(f(ext_b)), C.c_double(lam), C.c_double(td), abi.ptr(r),
                    abi.ptr(blk[0]), abi.ptr(blk[1]), abi.ptr(blk[2]), abi.ptr(blk[3]), abi.ptr(Jl), abi.ptr(Jt))
    for b in range(4):
        J[:rows, 7 * b:7 * b + 7] = blk[b].reshape(rows, 7)
    J[:rows, 28] = Jl[:rows]; J[:rows, 29] = Jt[:rows]
    return r, J, rows


def orc_loss(r, J, rows, delta):
    """orc_huber + orc_corrector as the oracle's minimiser applies them: (r', J', cost, Jacobian scale)."""
    from oracle import orc
    L = orc.lib()
    s = float(r[:rows] @ r[:rows])
    if delta <= 0:
        return r.copy(), J.copy(), 0.5 * s, 1.0
    rho = np.zeros(3)
    L.orc_huber(C.c_double(delta), C.c_double(s), abi.ptr(rho))
    rs = C.c_double(); sr = C.c_double(); asn = C.c_double()
    L.orc_corrector(abi.ptr(rho), C.c_double(s), C.byref(rs), C.byref(sr), C.byref(asn))
    rr = r.copy(); JJ = J.copy()
    rr[:rows] = rs.value * r[:rows]
    JJ[:rows] = sr.value * (J[:rows] - asn.value * np.outer(r[:rows], r[:rows] @ J[:rows]))
    return rr, JJ, 0.5 * rho[0], sr.value


def _cfg_values(cfg):
    c = abi.default_config(**cfg)
    return c.focal_length / 1.5, c.depth_sqrt_inf, c.huber_delta


def _raw_terms(pr, st, cfg):
    """Per observation (input order): type, block indices, r / J before the loss, rows."""
    s_px, s_d, _ = _cfg_values(cfg)
    out = []
    for (t, pi, pj, ea, eb, l), o in zip(_blocks(pr), pr["obs"]):
        g = lambda a, i: a[i] if i >= 0 else None   # noqa: E731
        r, J, rows = orc_obs_eval(t, o, g(st["pose"], pi), g(st["pose"], pj), g(st["ext"], ea), g(st["ext"], eb), st["lm"][l], st["td"], s_px, s_d)
        out.append(dict(t=t, blk=(pi, pj, ea, eb), lm=l, r=r, J=J, rows=rows))
    return out


def floors(J, ncol_segments):
    """Jb: |J| floored at the inf-norm of its own segment of the row; ncol_segments lists (start, width)."""
    Jb = np.abs(J).copy()
    for a, w in ncol_segments:
        seg = np.abs(J[..., a:a + w]).max(axis=-1, keepdims=True)
        Jb[..., a:a + w] = np.maximum(Jb[..., a:a + w], seg)
    return Jb


PROJ_SEGMENTS = [(7 * b + 3 * k, 3) for b in range(4) for k in range(2)] + [(7 * b + 6, 1) for b in range(4)] + [(28, 1), (29, 1)]
TRANSLATION = [0, 1, 2, 7, 8, 9, 14, 15, 16, 21, 22, 23]


def proj_floors(t, o, J, r, rows, lam, sc, s_px, s_d):
    """(Jb, rb) of one reprojection observation in the [pose_i 7 | pose_j 7 | ext_a 7 | ext_b 7 | lambda | td] layout.
    Pose and extrinsic entries are floored at their 3-column segment.  lambda, td and the residual are single entries
    that are differences of larger terms (a near-parallel bearing pair makes d r / d lambda small; r = s (B . (u_i - u_j))
    of two unit vectors), so they are floored at the magnitude of those terms: |J_t| / lambda^2 for lambda, s |v_j| +
    |J_t| |v_i| / |lambda| for td, and s for r, with J_t the row's largest translation entry and s the row's weight times
    the loss scale (for the depth rows: s_d times the larger inverse depth)."""
    Jb = floors(J, PROJ_SEGMENTS)
    rb = np.abs(r).copy()
    if t == abi.PROJ_DEPTH_PRIOR:
        rb[0] = max(rb[0], sc * s_d * max(abs(lam), 1.0 / float(o["depth"])))
        return Jb, rb
    jt = np.abs(J[:rows][:, TRANSLATION]).max(axis=1)
    il = 1.0 / max(abs(lam), 1e-300)
    vi, vj = float(np.abs(o["vel_i"]).max()), float(np.abs(o["vel_j"]).max())
    w = np.array([s_px, s_px, s_d * max(abs(lam), 1.0 / float(o["depth"]) if float(o["depth"]) else 0.0)])[:rows] * sc
    Jb[:rows, 28] = np.maximum(Jb[:rows, 28], jt * il * il)
    Jb[:rows, 29] = np.maximum(Jb[:rows, 29], w * vj + jt * vi * il)
    rb[:rows] = np.maximum(rb[:rows], w)
    return Jb, rb


def columns(pr):
    """Canonical (insertion-order) columns of the device's debug views: free poses, free extrinsics, td, speed-bias."""
    pc, ec = np.asarray(pr["pose_const"]).astype(bool), np.asarray(pr["ext_const"]).astype(bool)
    c = 0
    pose_col, ext_col = np.full(len(pc), -1), np.full(len(ec), -1)
    for i in range(len(pc)):
        if not pc[i]:
            pose_col[i] = c; c += 6
    for i in range(len(ec)):
        if not ec[i]:
            ext_col[i] = c; c += 6
    td_col = -1
    if not pr["td_const"]:
        td_col = c; c += 1
    nlc = c
    sb_col = nlc + 9 * np.arange(len(pr["sb_ids"]))
    return pose_col, ext_col, td_col, sb_col, nlc, nlc + 9 * len(pr["sb_ids"])


def proj_blocks(pr, st, cfg):
    """Loss-corrected per-observation terms of the reprojection factors, as arrays for ``assemble``."""
    _, _, delta = _cfg_values(cfg)
    pose_col, ext_col, td_col, _, _, _ = columns(pr)
    terms = _raw_terms(pr, st, cfg)
    M = len(terms)
    cols = np.full((M, 25), -1, np.int64); J = np.zeros((M, 3, 25)); Jb = np.zeros((M, 3, 25))
    r = np.zeros((M, 3)); Jl = np.zeros((M, 3)); Jlb = np.zeros((M, 3)); cost = np.zeros(M); rows = np.zeros(M, np.int64); lm = np.zeros(M, np.int64)
    s_px, s_d, _ = _cfg_values(cfg)
    rb = np.zeros((M, 3))
    for k, t in enumerate(terms):
        rr, JJ, c, sc = orc_loss(t["r"], t["J"], t["rows"], delta)
        JB, rb[k] = proj_floors(t["t"], pr["obs"][k], JJ, rr, t["rows"], st["lm"][t["lm"]], sc, s_px, s_d)
        pi, pj, ea, eb = t["blk"]
        if t["t"] != abi.PROJ_DEPTH_PRIOR:
            for b, (idx, tab) in enumerate(((pi, pose_col), (pj, pose_col), (ea, ext_col), (eb, ext_col))):
                if idx >= 0 and tab[idx] >= 0:
                    cols[k, 6 * b:6 * b + 6] = tab[idx] + np.arange(6)
            cols[k, 24] = td_col
        for b in range(4):
            J[k, :, 6 * b:6 * b + 6] = JJ[:, 7 * b:7 * b + 6]; Jb[k, :, 6 * b:6 * b + 6] = JB[:, 7 * b:7 * b + 6]
        J[k, :, 24] = JJ[:, 29]; Jb[k, :, 24] = JB[:, 29]
        r[k] = rr; Jl[k] = JJ[:, 28]; Jlb[k] = JB[:, 28]; cost[k] = c; rows[k] = t["rows"]; lm[k] = t["lm"]
    return dict(cols=cols, J=J, Jb=Jb, r=r, rb=rb, Jl=Jl, Jlb=Jlb, cost=cost, rows=rows, lm=lm)


def imu_blocks(pr, st):
    """IMU factor terms (orc_imu_eval, whitened) for windows that keep them."""
    from oracle import orc
    L = orc.lib()
    pose_col, _, _, sb_col, _, _ = columns(pr)
    pose = {int(f): i for i, f in enumerate(pr["frame_ids"])}
    sbi = {int(f): i for i, f in enumerate(pr["sb_ids"])}
    M = len(pr["imu"])
    cols = np.full((M, 30), -1, np.int64); J = np.zeros((M, 15, 30)); r = np.zeros((M, 15)); cost = np.zeros(M)
    g = abi.default_config().gravity_norm
    for k, m in enumerate(pr["imu"]):
        p = orc.OrcImuConst()
        p.sum_dt = float(m["sum_dt"]); p.delta_p[:] = m["delta_p"]; p.delta_q[:] = m["delta_q"]; p.delta_v[:] = m["delta_v"]
        p.linearized_ba[:] = m["linearized_ba"]; p.linearized_bg[:] = m["linearized_bg"]
        p.jacobian[:] = m["jacobian"].ravel(); p.covariance[:] = m["covariance"].ravel()
        si = np.zeros(225)
        assert L.orc_imu_sqrt_info(abi.ptr(np.ascontiguousarray(m["covariance"].ravel())), abi.ptr(si)) == 0
        p.sqrt_info[:] = si
        a, b = pose[int(m["frame_a"])], pose[int(m["frame_b"])]
        sa, sb = sbi[int(m["frame_a"])], sbi[int(m["frame_b"])]
        Js = [np.zeros((15, 7)), np.zeros((15, 9)), np.zeros((15, 7)), np.zeros((15, 9))]
        rr = np.zeros(15)
        x = [np.ascontiguousarray(v, dtype=np.float64) for v in (st["pose"][a], st["sb"][sa], st["pose"][b], st["sb"][sb])]
        L.orc_imu_eval(C.byref(p), C.c_double(g), abi.ptr(x[0]), abi.ptr(x[1]), abi.ptr(x[2]), abi.ptr(x[3]), abi.ptr(rr),
                       abi.ptr(Js[0]), abi.ptr(Js[1]), abi.ptr(Js[2]), abi.ptr(Js[3]))
        J[k] = np.concatenate([Js[0][:, :6], Js[1], Js[2][:, :6], Js[3]], axis=1)
        for off, c0, w in ((0, pose_col[a], 6), (6, sb_col[sa], 9), (15, pose_col[b], 6), (21, sb_col[sb], 9)):
            if c0 >= 0:
                cols[k, off:off + w] = c0 + np.arange(w)
        r[k] = rr; cost[k] = 0.5 * float(rr @ rr)
    Jb = floors(J, [(3 * i, 3) for i in range(10)])
    return dict(cols=cols, J=J, Jb=Jb, r=r, rb=np.abs(r), Jl=np.zeros((M, 15)), Jlb=np.zeros((M, 15)), cost=cost,
                rows=np.full(M, 15), lm=np.full(M, -1))


def assemble(blocks, n, nlc, nl):
    """Long-double sums of the terms and, per entry, the allowance 2 (C_J + m) eps sum Jb Jb."""
    out = {k: [np.zeros(s, LD), np.zeros(s, LD), np.zeros(s, np.int64)] for k, s in
           (("H", n * n), ("g", n), ("hl", nl), ("gl", nl), ("W", nl * nlc), ("cost", 1))}

    def add(key, idx, val, bnd, m):
        np.add.at(out[key][0], idx, val); np.add.at(out[key][1], idx, bnd); np.add.at(out[key][2], idx, m)
    for b in blocks:
        if len(b["cols"]) == 0:
            continue
        cols = b["cols"]; valid = cols >= 0
        J = np.where(valid[:, None, :], b["J"], 0).astype(LD); Jb = np.where(valid[:, None, :], b["Jb"], 0).astype(LD)
        r, rb, Jl, Jlb = b["r"].astype(LD), b["rb"].astype(LD), b["Jl"].astype(LD), b["Jlb"].astype(LD)
        rows = b["rows"]
        pair = valid[:, :, None] & valid[:, None, :]
        idx = (cols[:, :, None] * n + cols[:, None, :])[pair]
        mm = np.broadcast_to(rows[:, None, None], pair.shape)[pair]
        add("H", idx, np.einsum("kqa,kqb->kab", J, J)[pair], np.einsum("kqa,kqb->kab", Jb, Jb)[pair], mm)
        mv = np.broadcast_to(rows[:, None], valid.shape)[valid]
        add("g", cols[valid], np.einsum("kqa,kq->ka", J, r)[valid], np.einsum("kqa,kq->ka", Jb, rb)[valid], mv)
        has = b["lm"] >= 0
        if has.any():
            lm = b["lm"]
            add("hl", lm[has], np.einsum("kq,kq->k", Jl, Jl)[has], np.einsum("kq,kq->k", Jlb, Jlb)[has], rows[has])
            add("gl", lm[has], np.einsum("kq,kq->k", Jl, r)[has], np.einsum("kq,kq->k", Jlb, rb)[has], rows[has])
            wv = valid & has[:, None]
            add("W", (lm[:, None] * nlc + cols)[wv], np.einsum("kqa,kq->ka", J, Jl)[wv], np.einsum("kqa,kq->ka", Jb, Jlb)[wv],
                np.broadcast_to(rows[:, None], valid.shape)[wv])
        add("cost", np.zeros(len(rows), np.int64), b["cost"].astype(LD), 0.5 * np.einsum("kq,kq->k", rb, rb), np.ones(len(rows), np.int64))
    # the cost is one sum over every observation: m is the number of its terms
    out["cost"][2][:] = sum(len(b["rows"]) for b in blocks)
    return out


def reference_views(pr, st, cfg):
    _, _, _, _, nlc, n = columns(pr)
    blocks = [proj_blocks(pr, st, cfg)]
    if len(pr["imu"]):
        blocks.append(imu_blocks(pr, st))
    return assemble(blocks, n, nlc, len(pr["lm_ids"])), n, nlc


ITEMS = (("H", abi.DBG_HCC), ("g", abi.DBG_GC), ("hl", abi.DBG_HLL), ("gl", abi.DBG_GL), ("W", abi.DBG_W), ("cost", abi.DBG_COST))


def excess(dev, ref):
    """max over entries of |dev - sum| / allowance (an entry without terms must be exactly zero)."""
    val, bnd, m = ref
    tol = 2 * (LD(C_J) + m.astype(LD)) * LD(EPS) * bnd
    err = np.abs(np.asarray(dev, np.float64).astype(LD) - val)
    if np.any((tol == 0) & (err != 0)):
        return float("inf")
    nz = tol > 0
    return float(np.max(err[nz] / tol[nz], initial=0.0))


# ---------------------------------------------------------------------------------------------------------- CPU tests
def _routing(name, tpj=1):
    key = ("routing", name, tpj)
    if key not in _CACHE:
        _CACHE[key] = predict_routing(problem(name), tpj)
    return _CACHE[key]


def test_catalogue_reaches_every_variant():
    """Every instantiation is reached, and for each one some window routes most of its observations there."""
    V = abi.LIN_VARIANTS
    best = {v: 0.0 for v in V}
    for name in CATALOGUE:
        rt = _routing(name)
        tot = sum(rt[v]["obs"] for v in V)
        assert tot == len(problem(name)["obs"]), name
        for v in V:
            best[v] = max(best[v], rt[v]["obs"] / tot)
    assert all(b > 0.5 for b in best.values()), best
    # the cases the catalogue is built around
    assert _routing("mono_s0")[V[6]]["obs"] == len(problem("mono_s0")["obs"])
    assert _routing("mono_shift")[V[7]]["obs"] == len(problem("mono_shift")["obs"]) and _routing("mono_shift")["motion_needed"]
    assert not _routing("mono_s0")["motion_needed"]
    for name, pp in (("anchor_s0", V[4]), ("anchor_shift", V[5])):
        rt = _routing(name)
        assert rt[V[0]]["groups"] > 0 and rt[pp]["groups"] > 0 and rt[pp]["max_tiles_per_job"] == 1
        assert _routing(name, 8)[pp]["max_tiles_per_job"] == 4
    from test_ba_solve_shapes import predict_plan
    assert predict_plan(problem("stereo_ext"))["rec_stride"] == 32 and _routing("stereo_ext")[V[4]]["groups"] > 0
    assert _routing("stereo_ext")[V[0]]["groups"] > 0 and _routing("stereo_ext")[V[1]]["groups"] > 0
    assert predict_plan(problem("a2"))["n_leaf"] == 1 and predict_plan(problem("a2"))["rec_stride"] == 16
    assert _routing("a2")[V[4]]["groups"] > 0
    assert _routing("depth")[V[2]]["obs"] > 0 and _routing("depth")[V[0]]["obs"] == int(np.sum(problem("depth")["obs"]["type"] == abi.PROJ_DEPTH_PRIOR))
    assert _routing("depth_td")[V[3]]["obs"] > 0
    quad = problem("quad")["obs"]
    assert _routing("quad")[V[0]]["obs"] == int(np.sum(quad["type"] == abi.PROJ_1F2C)) > 0
    # the edge windows keep the routing of their plain counterparts
    assert _routing("mono_s0_edges")[V[6]]["obs"] == len(problem("mono_s0_edges")["obs"])
    assert _routing("anchor_shift_edges")[V[5]]["groups"] > 0 and _routing("stereo_td_edges")[V[1]]["obs"] == len(problem("stereo_td_edges")["obs"])


def test_bench_scale_handle_reaches_multi_tile_jobs():
    names, extra = bench_handle_layout(N_SM)
    prs = [problem(n) for n in names] + [bench(s) for s in extra]
    tpj = predict_tpj(prs, N_SM)
    assert tpj == 8
    V = abi.LIN_VARIANTS
    for v in V[4:]:
        assert any(predict_routing(p, tpj)[v]["max_tiles_per_job"] > 1 for p in prs[:len(names)] + [bench(False), bench(True)]), v


def _residual_norms(pr, cfg=None):
    return np.array([np.sqrt(np.sum(t["r"][:t["rows"]] ** 2)) for t in _raw_terms(pr, state_of_problem(pr), cfg or {})])


def test_catalogue_holds_every_edge_family():
    for name in ("mono_s0_edges", "anchor_shift_edges", "stereo_td_edges", "depth_edges"):
        pr = problem(name)
        for fam in EDGE_FAMILIES:
            assert len(pr["edges"][fam]) >= 1, (name, fam)
        nrm = _residual_norms(pr)
        assert np.sum(nrm > HUBER_DEFAULT) >= 10 and np.sum(nrm < HUBER_DEFAULT) >= 10, name
        assert nrm[pr["edges"]["outlier"]].min() > 10 * HUBER_DEFAULT, name
        assert np.any(pr["obs"]["pts_j"][:, 2] < 0) and np.any(pr["obs"]["pts_i"][:, 2] < 0)
        assert np.any(np.all(pr["obs"]["pts_j"] == (0.0, 0.0, 1.0), axis=1))
        assert (pr["poses"][:, 6] < 0).sum() >= 2 and pr["ext"][-1, 6] < 0
        assert pr["inv_dep"].min() < 0 and pr["inv_dep"].max() >= 10 and np.any(np.abs(pr["inv_dep"]) <= 1e-4)
    # fast-path and generic windows both carry the edges
    V = abi.LIN_VARIANTS
    assert _routing("mono_s0_edges")[V[6]]["obs"] > 0 and _routing("anchor_shift_edges")[V[5]]["obs"] > 0
    assert _routing("stereo_td_edges")[V[1]]["obs"] > 0 and _routing("depth_edges")[V[2]]["obs"] > 0
    # the 3-row factor and the depth prior in the Huber region
    pr = problem("depth_edges")
    nrm = _residual_norms(pr)
    for t in (abi.PROJ_2F1C_DEPTH, abi.PROJ_DEPTH_PRIOR):
        sel = pr["obs"]["type"] == t
        assert np.sum(nrm[sel] > HUBER_DEFAULT) >= 1 and np.sum(nrm[sel] < HUBER_DEFAULT) >= 1, t
    # huber_at: one residual within 1e-9 relative of delta
    for w in CONFIG_WINDOWS:
        d = config_of("huber_at", w)["huber_delta"]
        assert np.min(np.abs(_residual_norms(problem(w)) / d - 1)) <= 1e-9


# ---- the oracle against the reference's own classes
def ref_params(t, pose_i, pose_j, ext_a, ext_b, lam, td):
    lam, td = np.array([lam]), np.array([td])
    if t == abi.PROJ_2F2C:
        return [pose_i, pose_j, ext_a, ext_b, lam, td]
    if t == abi.PROJ_1F2C:
        return [ext_a, ext_b, lam, td]
    return [pose_i, pose_j, ext_a, lam, td]


# columns of each reference block in the oracle's [pose_i 7 | pose_j 7 | ext_a 7 | ext_b 7 | lambda | td] layout
REF_COLS = {abi.PROJ_2F1C: (0, 7, 14, 28, 29), abi.PROJ_2F2C: (0, 7, 14, 21, 28, 29), abi.PROJ_1F2C: (14, 21, 28, 29),
            abi.PROJ_2F1C_DEPTH: (0, 7, 14, 28, 29)}


def ref_obs_eval(t, o, pose_i, pose_j, ext_a, ext_b, lam, td, s_px, s_d, delta):
    """The reference's Evaluate (+ ResidualInfo's loss section) in the oracle's layout: (r (3), J (3 x 30), rows).  The
    depth prior (an autodiff functor, OneFrameDepth, depth_factor.h) is its one-line formula."""
    from oracle import ref
    r = np.zeros(3); J = np.zeros((3, 30))
    if t == abi.PROJ_DEPTH_PRIOR:
        rows = 1
        r[0] = (lam - 1.0 / float(o["depth"])) * s_d; J[0, 28] = s_d
    else:
        ref.configure(focal_length=1.5 * s_px, depth_sqrt_inf=s_d)
        rr, Js, _ = ref.proj_eval(t, o["pts_i"], o["pts_j"], o["vel_i"], o["vel_j"], float(o["td_i"]), float(o["td_j"]), float(o["depth"]),
                                  ref_params(t, pose_i, pose_j, ext_a, ext_b, lam, td))
        rows = len(rr)
        r[:rows] = rr
        for c0, Jk in zip(REF_COLS[t], Js):
            J[:rows, c0:c0 + Jk.shape[1]] = Jk
    if delta > 0:
        rr, JJ = ref.loss_correct(r[:rows], J[:rows], delta)
        r[:rows] = rr; J[:rows] = JJ
    return r, J, rows


def disagreement(t, o, x, cfgv, r_o, J_o, r_r, J_r, rows, sc):
    """Largest |oracle - reference| per entry in units of eps Jb (``proj_floors`` of the reference's values)."""
    Jb, rb = proj_floors(t, o, J_r, r_r, rows, x[4], sc, cfgv[0], cfgv[1])
    Jb, rb = Jb[:rows], rb[:rows]
    e = np.abs(J_o[:rows] - J_r[:rows]); er = np.abs(r_o[:rows] - r_r[:rows])
    q = [0.0]
    if np.any((Jb == 0) & (e != 0)) or np.any((rb == 0) & (er != 0)):
        return float("inf")
    q.append(float(np.max(e[Jb > 0] / (EPS * Jb[Jb > 0]), initial=0.0)))
    q.append(float(np.max(er[rb > 0] / (EPS * rb[rb > 0]), initial=0.0)))
    return max(q)


def edge_cases():
    """(window, config name, observation index) of every observation the edge families touch, each configuration."""
    out = []
    for name in ("mono_s0_edges", "anchor_shift_edges", "stereo_td_edges", "depth_edges"):
        idx = sorted(set(int(i) for fam in EDGE_FAMILIES for i in problem(name)["edges"][fam]))
        for cfg in ([None] + list(CONFIGS) if name in CONFIG_WINDOWS else [None]):
            out.extend((name, cfg, k) for k in idx)
    return out


def case_inputs(name, cfg_name, k):
    pr = problem(name); st = state_of_problem(pr)
    t, pi, pj, ea, eb, l = _blocks(pr)[k]
    s_px, s_d, delta = _cfg_values(config_of(cfg_name, name))
    g = lambda a, i: a[i] if i >= 0 else None   # noqa: E731
    return t, pr["obs"][k], (g(st["pose"], pi), g(st["pose"], pj), g(st["ext"], ea), g(st["ext"], eb), st["lm"][l], st["td"]), (s_px, s_d, delta)


def oracle_corrected(t, o, x, cfgv):
    s_px, s_d, delta = cfgv
    r, J, rows = orc_obs_eval(t, o, *x, s_px, s_d)
    rr, JJ, _, sc = orc_loss(r, J, rows, delta)
    return rr, JJ, rows, sc


def _ref_available():
    try:
        from oracle import ref
        return ref.available()
    except Exception:
        return False


needs_ref = pytest.mark.skipif(not _ref_available(), reason="oracle/_ref/libd2ref.so not built and no reference tree")


@needs_ref
def test_oracle_matches_reference_classes():
    """orc_proj_eval / the depth prior, orc_huber and the corrector at the catalogue's s_px, s_d and delta equal the
    reference's factor classes and loss section on every catalogue observation; the largest disagreement fixes C_J."""
    from oracle import ref
    worst = {}
    try:
        for name in CATALOGUE:
            pr = problem(name); st = state_of_problem(pr)
            cfgs = [None] + (list(CONFIGS) if name in CONFIG_WINDOWS else [])
            for cfg_name in cfgs:
                cfgv = _cfg_values(config_of(cfg_name, name))
                for k, (t, pi, pj, ea, eb, l) in enumerate(_blocks(pr)):
                    g = lambda a, i: a[i] if i >= 0 else None   # noqa: E731
                    x = (g(st["pose"], pi), g(st["pose"], pj), g(st["ext"], ea), g(st["ext"], eb), st["lm"][l], st["td"])
                    r_o, J_o, rows, sc = oracle_corrected(t, pr["obs"][k], x, cfgv)
                    r_r, J_r, rows_r = ref_obs_eval(t, pr["obs"][k], *x, *cfgv)
                    assert rows == rows_r
                    d = disagreement(t, pr["obs"][k], x, cfgv, r_o, J_o, r_r, J_r, rows, sc)
                    key = (name, cfg_name)
                    worst[key] = max(worst.get(key, 0.0), d)
    finally:
        ref.configure()
    m = max(worst.values())
    print("oracle vs reference, max |diff| / (eps Jb):", json.dumps({f"{a}/{b}": round(v, 2) for (a, b), v in worst.items()}))
    assert 4 * m <= C_J, (m, max(worst, key=worst.get))


def test_oracle_matches_frozen_reference_edges():
    """The same comparison on the frozen reference values of the edge observations (tests/golden/ref_lin_edges.npz)."""
    g = np.load(GOLD)
    cases = edge_cases()
    assert len(cases) == len(g["r"]) and 0 < len(cases) <= 1000
    worst = 0.0
    for i, (name, cfg_name, k) in enumerate(cases):
        t, o, x, cfgv = case_inputs(name, cfg_name, k)
        assert int(g["typ"][i]) == t and np.array_equal(g["cfg"][i], np.array(cfgv))
        r_o, J_o, rows, sc = oracle_corrected(t, o, x, cfgv)
        worst = max(worst, disagreement(t, o, x, cfgv, r_o, J_o, g["r"][i], g["J"][i], rows, sc))
    assert 4 * worst <= C_J, worst


def test_criterion_is_sharp():
    """A Jacobian entry moved by 1e-8 of its segment, or one observation's residual scaled by 1 + 1e-5, breaks the
    allowance of the entries it feeds."""
    pr = problem("mono_s0_edges"); st = state_of_problem(pr)
    b = proj_blocks(pr, st, {})
    _, _, _, _, nlc, n = columns(pr)
    ref = assemble([b], n, nlc, len(pr["lm_ids"]))
    bad = dict(b); bad["J"] = b["J"].copy()
    k = int(np.argmax(b["Jb"][:, 0, 3]))
    bad["J"][k, 0, 3] += 1e-8 * b["Jb"][k, 0, 3]
    dev = assemble([bad], n, nlc, len(pr["lm_ids"]))
    H = dev["H"][0].astype(np.float64)
    assert excess(H, ref["H"]) > 1.0 and excess(ref["H"][0].astype(np.float64), ref["H"]) <= 1.0
    bad = dict(b); bad["r"] = b["r"].copy(); bad["r"][k] *= 1 + 1e-5
    g = assemble([bad], n, nlc, len(pr["lm_ids"]))["g"][0].astype(np.float64)
    assert excess(g, ref["g"]) > 1.0


# ---------------------------------------------------------------------------------------------------------- GPU tests
def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _record(**vals):
    """Appends measured ratios to the JSON-lines file D2BA_LIN_LOG names (the DESIGN.md table)."""
    path = os.environ.get("D2BA_LIN_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(vals) + "\n")


def check_window(s, w, pr, cfg, label, routing=None):
    """Entry-wise check of one window of a linearised handle at the device's own state; returns the worst ratio."""
    st = state_of_device(s, w, pr)
    ref, n, nlc = reference_views(pr, st, cfg)
    assert int(s.debug_get(w, abi.DBG_N_CAM, np.int64)[0]) == n and int(s.debug_get(w, abi.DBG_N_LC, np.int64)[0]) == nlc
    ratios = {}
    for key, item in ITEMS:
        ratios[key] = excess(s.debug_get(w, item), ref[key])
    rt = routing or s.debug_lin_jobs(w)
    _record(label=label, ratios=ratios, variants=[v for v in abi.LIN_VARIANTS if rt[v]["obs"]])
    assert max(ratios.values()) <= 1.0, (label, ratios)
    return ratios


def _handle(names_prs, cfg=None):
    from d2slam_b200.solver import Solver
    s = Solver(max_windows=len(names_prs), **(cfg or {}))
    for i, pr in enumerate(names_prs):
        load(pr, s, i)
    s.finalize()
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_window_alone(name):
    pr = problem(name)
    s = _handle([pr])
    assert s.debug_lin_jobs(0) == predict_routing(pr, predict_tpj([pr], _n_sm()))
    s.debug_linearize()
    check_window(s, 0, pr, {}, f"{name}/alone/linearize")
    s.solve_fixed(3)
    s.debug_linearize()
    check_window(s, 0, pr, {}, f"{name}/alone/solve3")
    # a fresh handle's first iteration evaluates the cost on the solve path's tiles (no motion upload)
    s = _handle([pr])
    rep = s.solve_fixed(1)[0]
    ref, _, _ = reference_views(pr, state_of_problem(pr), {})
    assert excess(np.array([rep.initial_cost]), ref["cost"]) <= 1.0, (name, rep.initial_cost, float(ref["cost"][0][0]))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", list(CONFIGS))
@pytest.mark.parametrize("name", CONFIG_WINDOWS)
def test_window_configurations(name, cfg_name):
    pr = problem(name)
    cfg = config_of(cfg_name, name)
    s = _handle([pr], cfg)
    s.debug_linearize()
    check_window(s, 0, pr, cfg, f"{name}/{cfg_name}/linearize")
    s.solve_fixed(3)
    s.debug_linearize()
    check_window(s, 0, pr, cfg, f"{name}/{cfg_name}/solve3")


@pytest.mark.gpu
def test_mixed_handle():
    names = list(CATALOGUE)
    prs = [problem(n) for n in names]
    s = _handle(prs)
    tpj = predict_tpj(prs, _n_sm())
    for i, name in enumerate(names):
        assert s.debug_lin_jobs(i) == predict_routing(prs[i], tpj), name
    s.debug_linearize()
    for i, name in enumerate(names):
        check_window(s, i, prs[i], {}, f"{name}/mixed/linearize")
    s.solve_fixed(3)
    s.debug_linearize()
    for i, name in enumerate(names):
        check_window(s, i, prs[i], {}, f"{name}/mixed/solve3")


def bench_handle_layout(n_sm):
    """The catalogue plus bench windows (both td-stamp variants, alternating) until the handle reaches 8 tiles per job."""
    names = list(CATALOGUE)
    prs = [problem(n) for n in names]
    extra = []
    b = [bench(False), bench(True)]
    while predict_tpj(prs + [b[i % 2] for i in range(len(extra))], n_sm) < 8:
        extra.append(len(extra) % 2 == 1)
    return names, extra


@pytest.mark.gpu
def test_bench_scale_handle():
    """Multi-tile jobs: the cross-tile accumulation and the next tile's prefetch in every fast-path instantiation."""
    n_sm = _n_sm()
    names, extra = bench_handle_layout(n_sm)
    b = [bench(False), bench(True)]
    prs = [problem(n) for n in names] + [b[int(e)] for e in extra]
    s = _handle(prs)
    tpj = predict_tpj(prs, n_sm)
    assert tpj == 8
    multi = {v: 0 for v in abi.LIN_VARIANTS[4:]}
    for i, pr in enumerate(prs):
        rt = s.debug_lin_jobs(i)
        if i < len(names) + 2:
            assert rt == predict_routing(pr, tpj), i
        for v in multi:
            multi[v] = max(multi[v], rt[v]["max_tiles_per_job"])
    assert all(m > 1 for m in multi.values()), multi
    checked = list(range(len(names))) + list(range(len(names), min(len(prs), len(names) + 8)))
    s.debug_linearize()
    for i in checked:
        check_window(s, i, prs[i], {}, f"{names[i] if i < len(names) else 'bench'}/bench_handle/linearize")
    s.solve_fixed(3)
    s.debug_linearize()
    for i in checked:
        check_window(s, i, prs[i], {}, f"{names[i] if i < len(names) else 'bench'}/bench_handle/solve3")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mono_s0", "mono_s0_edges"])
def test_td_transition_refinalizes_into_the_shift_path(name):
    """td constant and equal to the stamps (pp<true,*>), then td set to another constant: the handle re-finalizes into
    pp<false,*> with the motion halves uploaded, and passes the same checks."""
    pr = problem(name)
    s = _handle([pr])
    V = abi.LIN_VARIANTS
    rt = s.debug_lin_jobs(0)
    assert rt[V[6]]["obs"] == len(pr["obs"]) and rt["motion_needed"] == 0
    s.solve_fixed(2)
    s.set_blocks(0, abi.TD, np.zeros(1, np.int64), np.array([0.0015]), np.array([1], np.uint8))
    s.finalize()
    rt = s.debug_lin_jobs(0)
    assert rt[V[7]]["obs"] == len(pr["obs"]) and rt["motion_needed"] == 1
    pr2 = dict(pr); pr2["td"] = 0.0015
    assert rt == predict_routing(synth.Problem(pr2), 1)
    s.debug_linearize()
    check_window(s, 0, pr, {}, f"{name}/transition/linearize")
    s.solve_fixed(2)
    s.debug_linearize()
    check_window(s, 0, pr, {}, f"{name}/transition/solve2")
