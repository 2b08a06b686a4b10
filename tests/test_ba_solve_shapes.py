"""BA reduced-camera solve at every boundary of the window plan d2ba_finalize chooses.

d2ba_finalize picks, per window, among about a dozen solve paths from size thresholds and structural tests (fused one-CTA
solve, one-CTA or tiled Schur complement, speed-bias elimination, leaf elimination, shared-memory or global Cholesky, 96-,
128- or 256-byte landmark records and their gathers).  ``predict_plan`` restates those rules from the problem alone; the
catalogue below puts windows on both sides of every rule, and a CPU test proves that it does.  On the GPU every catalogue
window is checked alone in a handle and again in one mixed handle that holds all of them at once:

- the plan the library reports (D2BA_DBG_PLAN) equals ``predict_plan``;
- the normal equations equal the CPU oracle's;
- the device-formed Schur complement equals a long-double assembly from the device's own views, entry by entry within
  2 n eps times the sum of the magnitudes of the entry's terms;
- the Gauss-Newton step has a normwise backward error on the full damped system that is at most max(floor, 10 x that of
  a float64 numpy solve in the same elimination order);
- the first dogleg step and 8 fixed iterations match the oracle.
"""
import json
import os

import numpy as np
import pytest

from d2slam_b200 import abi, synth
from helpers import relerr, state_diff, state_of

MU0 = 1e-8                 # LM regularisation of the GN step after d2ba_debug_linearize (SolverParams::mu0)
SMEM_OPTIN = 232448        # H100 cudaDevAttrMaxSharedMemoryPerBlockOptin (227 KB)
ETA_FLOOR = 1e-16          # H100 (700 W): device eta <= 2.7e-17 over the catalogue, DESIGN.md section 4


# ---------------------------------------------------------------------------------------------------------- shared memory
# restated from d2slam_b200/csrc/d2ba_launch.cuh and d2ba_kernels.cu; the GPU tests compare every decision that depends on them
def chol_smem_bytes(n):                 # d2ba_launch.cuh: chol_smem_bytes (kCsNB = 8)
    pr, need = 8 * ((n + 2) & ~1), n + 1 + 16 * 32
    return ((n + 1) * ((n + 1) & ~1) + ((n + 1) & ~1) + max(pr, need)) * 8 + 32


def sbe_smem_bytes(ldw, n_c, nb):       # d2ba_launch.cuh: sbe_smem_bytes (kSeSlotRows = 9)
    return (3 * 9 * ldw + nb * 2 * 81 + nb * 9 + n_c + 9 * nb + 16) * 8


def sb_back_smem_bytes(nlc, nb):        # d2ba_launch.cuh: sb_back_smem_bytes
    return (((nlc + 31) & ~31) + 9 * nb + 171 * nb) * 8


def leaf_elim_smem_bytes(n, nh):        # d2ba_launch.cuh: leaf_elim_smem_bytes, leaf_lda (kLeafLmChunk = 16)
    n1 = n + nh + 1
    return (n1 * (n | 1) + ((n + 1) & ~1) + 8 * ((n1 + 1) & ~1) + 64 + 16 * n1 + 8) * 8


def solve_small_fits(ldw):              # d2ba_launch.cuh: solve_small_fits (kSolveMaxB = 12, 4 warps)
    nb8 = ldw // 8
    return nb8 * (nb8 + 1) // 2 <= 12 * 4


def chol_global_smem_bytes(max_rows):   # d2ba_kernels.cu: chol_glob_smem_bytes (kNB = 32)
    return (32 * (max_rows + 4) + 2 * max_rows + 16 + 16 * 32 + 32 * 33) * 8


def gather_smem_bytes(max_ldw):         # d2ba_kernels.cu: gather_smem_bytes (kGatherWarps = 8, kG16Lm = 16)
    return max(8 * max_ldw * 8, 16 * max_ldw * 8)


def roundup(v, m):
    return (v + m - 1) // m * m


# ---------------------------------------------------------------------------------------------------------- the plan
def _indices(pr):
    pose = {int(f): i for i, f in enumerate(pr["frame_ids"])}
    ext = {int(c): i for i, c in enumerate(pr["cam_ids"])}
    sb = {int(f): i for i, f in enumerate(pr["sb_ids"])}
    lm = {int(l): i for i, l in enumerate(pr["lm_ids"])}
    obs = []
    for o in pr["obs"]:
        t = int(o["type"])
        pi = pj = ea = eb = -1
        if t != abi.PROJ_DEPTH_PRIOR:
            ea = ext[int(o["cam_a"])]
            if t in (abi.PROJ_2F2C, abi.PROJ_1F2C):
                eb = ext[int(o["cam_b"])]
            if t != abi.PROJ_1F2C:
                pi, pj = pose[int(o["frame_a"])], pose[int(o["frame_b"])]
        obs.append((t, pi, pj, ea, eb, lm[int(o["landmark_id"])]))
    imu = [(pose[int(m["frame_a"])], sb[int(m["frame_a"])], pose[int(m["frame_b"])], sb[int(m["frame_b"])]) for m in pr["imu"]]
    return obs, imu


def predict_plan(pr):
    """Pass A of d2ba_finalize (d2ba_host.cu) restated for one window: the D2BA_DBG_PLAN fields that do not depend on the
    other windows of the handle (fused_solve before the handle-wide gate, chol_threads left to ``predict_handle``).
    Speed-bias blocks are all free (Problem.load), td is present."""
    obs, imu = _indices(pr)
    np_, ne, nsb, nl = len(pr["frame_ids"]), len(pr["cam_ids"]), len(pr["sb_ids"]), len(pr["lm_ids"])
    pc, ec = np.asarray(pr["pose_const"]).astype(bool), np.asarray(pr["ext_const"]).astype(bool)
    td_free = not pr["td_const"]
    nlc_cnt = 6 * (int((~pc).sum()) + int((~ec).sum())) + int(td_free)
    # speed-bias elimination: a block-tridiagonal chain of at most kSeMaxBlocks = 32 blocks
    nb = nsb
    sb_ok = nb >= 1 and nlc_cnt >= 1 and all(abs(si - sj) <= 1 for _, si, _, sj in imu) and nb <= 32
    prior_poses = [] if pr.get("prior") is None else [int(r["id"]) for r in pr["prior"][2] if int(r["kind"]) == abi.POSE]
    prior_idx = [list(map(int, pr["frame_ids"])).index(f) for f in prior_poses]
    # leaves: components (through shared landmarks) of the free poses no IMU factor or prior touches
    leaves = []
    if sb_ok and nlc_cnt + 1 > 96:
        hub = np.zeros(np_, bool)
        for pi, _, pj, _ in imu:
            hub[pi] = hub[pj] = True
        hub[prior_idx] = True
        uf = list(range(np_))

        def find(x):
            while uf[x] != x:
                uf[x] = uf[uf[x]]; x = uf[x]
            return x
        first = [-1] * nl
        for t, pi, pj, _, _, l in obs:
            for pz in (pi, pj):
                if pz < 0 or hub[pz] or pc[pz]:
                    continue
                if first[l] < 0:
                    first[l] = pz; continue
                a, b = find(pz), find(first[l])
                if a != b:
                    uf[max(a, b)] = min(a, b)
        comp = {}
        for i in range(np_):
            if hub[i] or pc[i]:
                continue
            r = find(i)
            if r not in comp:
                comp[r] = len(leaves); leaves.append([])
            leaves[comp[r]].append(i)
        n_hub_cols = nlc_cnt - sum(6 * len(lf) for lf in leaves)
        kept = []
        for lf in leaves:
            nl6 = 6 * len(lf)
            if nl6 <= 96 and n_hub_cols >= 1 and leaf_elim_smem_bytes(nl6, n_hub_cols) <= 200 * 1024:
                kept.append(lf)
            else:
                n_hub_cols += nl6
        leaves = [] if (not kept or n_hub_cols > 3 * nlc_cnt // 4) else kept
    # columns: [leaf 0 | leaf 1 | ... | hub poses | extrinsics | td | speed-bias]
    pose_col, ext_col, c = [-1] * np_, [-1] * ne, 0
    leaf_of = [-1] * np_
    for li, lf in enumerate(leaves):
        for i in lf:
            pose_col[i] = c; c += 6; leaf_of[i] = li
    hub0 = c
    for i in range(np_):
        if not pc[i] and leaf_of[i] < 0:
            pose_col[i] = c; c += 6
    for i in range(ne):
        if not ec[i]:
            ext_col[i] = c; c += 6
    td_col = c if td_free else -1
    c += int(td_free)
    n_lc = c
    sb_col = [n_lc + 9 * i for i in range(nsb)]
    n_c = n_lc + 9 * nsb
    n_hub, n_leaf = n_lc - hub0, len(leaves)
    ldw = roundup(n_lc + 1, 8)
    # pair-major groups, their slots, the landmark tile masks and the Hcc pattern
    groups = {}
    for k, o in enumerate(obs):
        groups.setdefault(o[:5], []).append(k)
    mask = [1 << (n_lc // 32)] * nl
    hpat = np.zeros((n_c, n_c), bool)

    def hblock(ra, rs, ca, cs):
        if ra >= 0 and ca >= 0:
            hpat[ra:ra + rs, ca:ca + cs] = True; hpat[ca:ca + cs, ra:ra + rs] = True
    any_wide, all_pp, n_tile, slot0, slot1 = False, True, 0, [], []
    for key in sorted(groups):
        t, pi, pj, ea, eb = key
        members = groups[key]
        cols = [pose_col[pi] if pi >= 0 else -1, pose_col[pj] if pj >= 0 else -1, ext_col[ea] if ea >= 0 else -1, ext_col[eb] if eb >= 0 else -1]
        if t == abi.PROJ_DEPTH_PRIOR:
            cols = [-1] * 4
        src = [s for s in range(4) if cols[s] >= 0]
        scol = [cols[s] for s in src]
        gtd = -1 if t == abi.PROJ_DEPTH_PRIOR else td_col
        nct = 2 if (len(scol) <= 2 and gtd < 0) else 4
        rows = 3 if t == abi.PROJ_2F1C_DEPTH else (1 if t == abi.PROJ_DEPTH_PRIOR else 2)
        any_wide |= nct == 4
        pp = (nct == 2 and rows == 2 and not any(s >= 2 for s in src) and t in (abi.PROJ_2F1C, abi.PROJ_2F2C)
              and src == [0, 1])
        all_pp &= pp
        n_tile += (len(members) + 31) // 32
        for a in range(len(scol)):
            for b in range(a + 1):
                hblock(scol[a], 6, scol[b], 6)
            if gtd >= 0:
                hblock(gtd, 1, scol[a], 6)
        if gtd >= 0:
            hblock(gtd, 1, gtd, 1)
        for k in members:
            l = obs[k][5]
            for col, wd in [(sc, 6) for sc in scol] + ([(gtd, 1)] if gtd >= 0 else []):
                mask[l] |= (1 << (col // 32)) | (1 << ((col + wd - 1) // 32))
            slot0.append((l, scol[0] if scol else -1)); slot1.append((l, scol[1] if len(scol) > 1 else -1))
    s0 = {}
    clash = False
    for l, c0 in slot0:
        if c0 >= 0:
            clash |= s0.setdefault(l, c0) != c0
    clash |= any(c1 >= 0 and s0.get(l) == c1 for l, c1 in slot1)
    gather_nosync = 0 if clash else 1
    row_tiles = n_lc // 32 + 1 if not leaves else max([1] + [bin(m).count("1") for m in mask])
    rec_stride, n_g12 = (32 if any_wide else 16), 0
    if not any_wide and all_pp and n_leaf == 0 and gather_nosync:
        cnt = np.bincount([o[5] for o in obs], minlength=nl)
        if cnt.max(initial=0) <= 32 and len(set(slot1)) == len(slot1):
            rec_stride, l = 12, 0
            while l < nl:
                l0, r = l, 0
                while l < nl and l - l0 < 31 and r + cnt[l] <= 32:
                    r += cnt[l]; l += 1
                n_g12 += 1
    schur_small = int(n_lc + 1 <= 96)
    hub_small = int(n_leaf > 0 and n_hub + 1 <= 96)
    ok = sb_ok and (sbe_smem_bytes(roundup(n_hub + 1, 8), n_c, nb) <= 200 * 1024 and sb_back_smem_bytes(n_hub, nb) <= 200 * 1024)
    ndense = n_hub if (ok or n_leaf > 0) else n_c
    chol_smem = int(n_c >= 1 and chol_smem_bytes(ndense) <= SMEM_OPTIN - 16)
    fused = int(n_leaf == 0 and ok and schur_small and chol_smem and solve_small_fits(ldw))
    wt_rows = roundup(max(nl + (9 * nb if ok else 0) + 6 * sum(len(lf) for lf in leaves), 1), 32)
    # the rest of the Hcc pattern: IMU factors and the prior (consensus off in this catalogue)
    for pi, si, pj, sj in imu:
        bc, bs = [pose_col[pi], sb_col[si], pose_col[pj], sb_col[sj]], [6, 9, 6, 9]
        for a in range(4):
            for b in range(a + 1):
                hblock(bc[a], bs[a], bc[b], bs[b])
    for i in prior_idx:
        hblock(pose_col[i], 6, pose_col[i], 6)
    schur = [0, 0]
    if not schur_small:
        ntw, nchunk = (n_lc + 1 + 31) // 32, wt_rows // 32
        cmask = [0] * nchunk
        for l in range(nl):
            cmask[l // 32] |= mask[l]
        hubmask = sum(1 << t for t in range(hub0 // 32, n_lc // 32 + 1))
        for r in range(nl, wt_rows):
            cmask[r // 32] |= hubmask
        lm_chunks = (nl + 31) // 32
        low = np.tril(hpat[:n_lc, :n_lc])
        tpat = np.zeros((ntw, ntw), bool)
        rr, cc = np.nonzero(low)
        tpat[rr // 32, cc // 32] = True
        for stage in (0, 1):
            for tm in range(ntw if n_lc > 0 else 0):
                for tn in range(tm + 1):
                    in_hub = tm * 32 + 31 >= hub0 and tn * 32 + 31 >= hub0
                    has_leaf = tn * 32 < hub0
                    if (not has_leaf) if stage == 0 else (not in_hub or hub_small):
                        continue
                    kend = lm_chunks if stage == 0 else nchunk
                    cn = sum(1 for kc in range(kend) if (cmask[kc] >> tm) & 1 and (cmask[kc] >> tn) & 1)
                    if cn == 0 and not tpat[tm, tn] and tm != ntw - 1:
                        continue
                    schur[stage] += 1
        if not ok:
            schur[1] += sum(tm + 1 for tm in range(n_lc // 32, n_c // 32 + 1))
    plan = dict(fused_solve=fused, schur_small=schur_small, hub_small=hub_small, chol_smem=chol_smem, chol_threads=0,
                sb_elim=int(ok), n_sbe=nb, n_leaf=n_leaf, hub0=hub0, n_hub=n_hub, n_lc=n_lc, n_c=n_c, ldw=ldw,
                rec_stride=rec_stride, gather_nosync=gather_nosync, row_tiles=row_tiles, n_g12=n_g12, n_tile=n_tile,
                schur0=schur[0], schur1=schur[1])
    assert set(plan) == set(abi.PLAN_FIELDS)
    return plan


def predict_handle(plans, n_sm):
    """The handle-wide rules of d2ba_finalize on top of ``predict_plan``: k_solve_small only with at least 3 eligible
    windows per SM (kFusedMinWindowsPerSM), one k_chol_smem thread count from the largest shared-memory system, and the
    refusal (code 23) of a k_chol or gather row buffer beyond the device's shared memory.  -> (plans, refusal code)"""
    plans = [dict(p) for p in plans]
    if sum(p["fused_solve"] for p in plans) < 3 * n_sm:
        for p in plans:
            p["fused_solve"] = 0
    dense = [(p["n_hub"] if (p["sb_elim"] or p["n_leaf"]) else p["n_c"], p) for p in plans]
    max_n_smem = max([n for n, p in dense if p["chol_smem"]], default=0)
    launched = any(p["chol_smem"] and not p["fused_solve"] for p in plans)
    for p in plans:
        p["chol_threads"] = (128 if max_n_smem <= 96 else 512) if launched else 0
    max_rows = max([n + 1 for n, p in dense if not p["chol_smem"]], default=1)
    refusal = 0
    if any(p["n_lc"] // 32 >= 64 for p in plans):
        refusal = 27
    elif chol_global_smem_bytes(max(max_rows, 2)) > SMEM_OPTIN - 16 or gather_smem_bytes(32 * max(p["row_tiles"] for p in plans)) > SMEM_OPTIN:
        refusal = 23
    return plans, refusal


# ---------------------------------------------------------------------------------------------------------- catalogue
def _window(seed, n_frames, n_landmarks=40, **kw):
    return synth.make_window(seed=seed, n_frames=n_frames, n_landmarks=n_landmarks, **kw)


def _remote(seed, n_agents, n_frames, n_landmarks=None, shared=10):
    pr = synth.make_swarm(seed=seed, n_agents=n_agents, n_frames=n_frames, only_agents=[0], shared_per_pair=shared,
                          n_landmarks=n_landmarks or max(60, (n_agents - 1) * shared + 10))[0]
    pr["consensus"] = None
    return pr


def _extra_imu(pr, a, b):
    """One more IMU factor between frames a and b (breaks the block-tridiagonal speed-bias chain)."""
    m = pr["imu"][a:a + 1].copy()
    m["frame_a"], m["frame_b"] = pr["frame_ids"][a], pr["frame_ids"][b]
    pr["imu"] = np.concatenate([pr["imu"], m])
    return pr


def _few_remote_free(pr, n_free):
    pc = pr["pose_const"].copy(); pc[pr["n_own"] + n_free:] = 1; pr["pose_const"] = pc
    return pr


def _const_anchor(seed, n_frames):
    return _window(seed, n_frames, with_prior=False)            # frame 0 constant


def _depth(seed):
    pr = _window(seed, 6, 60)
    ids, tptr, tobs = pr["tracks"]
    tobs = tobs.copy(); tobs["depth_mea"] = 1
    pr["obs"] = synth.tracks_to_obs(ids, tptr, tobs, fuse_dep=True, min_d=0.3, max_d=50.0)
    return pr


def _degenerate(seed):
    """Two consecutive constant poses inside the speed-bias chain (frames 2 and 3; the anchor frame 0 is constant too), a
    landmark seen only from constant poses (zero row of W), a landmark with one record, and a free pose that no landmark
    sees (frame 5)."""
    pr = _window(seed, 6, 30, with_prior=False)
    pc = pr["pose_const"].copy(); pc[[0, 2, 3]] = 1; pr["pose_const"] = pc
    f, o = pr["frame_ids"], pr["obs"]
    lm0, lm1 = pr["lm_ids"][0], pr["lm_ids"][1]
    keep = ((o["frame_b"] != f[5]) & ((o["landmark_id"] != lm0) | np.isin(o["frame_b"], f[[2, 3]]))
            & ((o["landmark_id"] != lm1) | (o["frame_b"] == f[4])))
    pr["obs"] = o[keep]
    return pr


def _no_1f2c(pr):
    """Drop the anchor frame's second-camera observations: 2F - 2 records per landmark in a stereo window."""
    pr["obs"] = pr["obs"][pr["obs"]["type"] != abi.PROJ_1F2C]
    return pr


CATALOGUE = {
    # fused one-CTA solve: ldw = roundup(n_lc + 1, 8) <= 72
    "f11": lambda: _window(101, 11),
    "f11_td": lambda: _window(102, 11, estimate_td=True, td_offset=0.002),
    "f12": lambda: _window(103, 12),
    "f11_stereo_ext": lambda: _window(104, 11, cams="stereo", estimate_extrinsic=True),
    # k_schur_small: n_lc + 1 <= 96
    "f15_td": lambda: _window(105, 15, estimate_td=True, td_offset=0.002),
    "f16": lambda: _window(106, 16),
    # shared-memory Cholesky of the pose part after the speed-bias elimination
    "f27": lambda: _window(107, 27),
    "f28": lambda: _window(108, 28),
    # speed-bias elimination: <= 32 blocks in a chain
    "f32": lambda: _window(109, 32),
    "f33": lambda: _window(110, 33),
    "f12_imu_2_4": lambda: _extra_imu(_window(111, 12), 2, 4),
    # k_chol: the largest n_c whose panel fits the shared memory (one frame more is refused)
    "f53": lambda: _window(112, 53, 30),
    # leaves: <= 96 columns and leaf_elim_smem_bytes <= 200 KB; hub <= 3/4 n_lc; hub_small: n_hub + 1 <= 96
    "a2_f15": lambda: _remote(113, 2, 15),
    "a2_f16": lambda: _remote(114, 2, 16),
    "a2_f17": lambda: _remote(115, 2, 17),
    "a2_f15_two_remote_free": lambda: _few_remote_free(_remote(116, 2, 15), 2),
    # 96-byte records: <= 32 records per landmark; k_lm_gather12 chunks of <= 31 landmarks / 32 records
    "f2_lm40": lambda: _window(117, 2, 40),
    "f17": lambda: _window(118, 17),
    "f34": lambda: _window(119, 34),
    # k_lm_gather16 with the record barrier (constant anchor: gather_nosync = 0), 16 / 17 / 32 / 33 records
    "anchor_const_f17": lambda: _const_anchor(120, 17),
    "anchor_const_f18": lambda: _const_anchor(121, 18),
    "anchor_const_f33": lambda: _const_anchor(122, 33),
    "anchor_const_f34": lambda: _const_anchor(123, 34),
    # k_lm_gather (256-byte records): stereo with td free, 17 and 33 records per landmark
    "stereo_td_f9": lambda: _window(124, 9, cams="stereo", estimate_td=True, td_offset=0.002),
    "stereo_td_f17": lambda: _window(125, 17, cams="stereo", estimate_td=True, td_offset=0.002),
    "stereo_td_f9_no1f2c": lambda: _no_1f2c(_window(126, 9, cams="stereo", estimate_td=True, td_offset=0.002)),
    "stereo_td_f17_no1f2c": lambda: _no_1f2c(_window(127, 17, cams="stereo", estimate_td=True, td_offset=0.002)),
    # 32-observation tiles: 1, 31, 32, 33, 64, 65 landmarks per pose pair
    **{f"f2_lm{n}": (lambda n=n: _window(126 + n, 2, n)) for n in (1, 31, 32, 33, 64, 65)},
    # factor variants
    "depth": lambda: _depth(200),
    "quad": lambda: _window(201, 6, 100, cams="quad"),
    # degenerate structure
    "degenerate": lambda: _degenerate(202),
}
# refused by d2ba_finalize, or too large for the mixed handle and the oracle's fixed schedule
LARGE = {
    "f54": (lambda: _window(130, 54, 30), 23),
    "a31_f11": (lambda: _remote(131, 31, 11, 320), 0),
    "a32_f11": (lambda: _remote(132, 32, 11, 330), 27),
}
# the message of each refusal: the k_chol panel (configure_launches), the landmark tile masks
REFUSAL_MESSAGE = {
    "f54": r"rc=23: cudaFuncSetAttribute failed \(shared memory request too large\?\)",
    "a32_f11": r"rc=27: finalize: window 0 has 2112 landmark-coupled columns",
}

_CACHE = {}


def problem(name):
    if name not in _CACHE:
        _CACHE[name] = CATALOGUE[name]() if name in CATALOGUE else LARGE[name][0]()
    return _CACHE[name]


def plan_of(name):
    key = ("plan", name)
    if key not in _CACHE:
        _CACHE[key] = predict_plan(problem(name))
    return _CACHE[key]


def records_per_landmark(pr):
    lm = {int(l): i for i, l in enumerate(pr["lm_ids"])}
    return np.bincount([lm[int(l)] for l in pr["obs"]["landmark_id"]], minlength=len(lm))


def landmarks_per_pair(pr):
    keys = {}
    for o in pr["obs"]:
        k = (int(o["type"]), int(o["frame_a"]), int(o["frame_b"]), int(o["cam_a"]), int(o["cam_b"]))
        keys[k] = keys.get(k, 0) + 1
    return sorted(keys.values())


# ---------------------------------------------------------------------------------------------------------- references
def damped_views(get, n, nlc, nl):
    """(Hd, g, W, hp, gl) of the damped system the GN step solves, from DBG_* views in canonical order; D as in the
    oracle (sqrt of the diagonal, clamped to [1e-6, 1e32])."""
    H = get(abi.DBG_HCC).reshape(n, n); g = get(abi.DBG_GC)
    hl = get(abi.DBG_HLL); gl = get(abi.DBG_GL); W = get(abi.DBG_W).reshape(nl, nlc)
    d2c = np.clip(np.sqrt(np.diag(H)), 1e-6, 1e32) ** 2
    d2l = np.clip(np.sqrt(hl), 1e-6, 1e32) ** 2
    Hd = H + np.diag(MU0 * d2c)
    return Hd, g, W, hl + MU0 * d2l, gl


def schur_excess(S_dev, Hd, W, hp):
    """max over the landmark-coupled entries of |S_dev - S| / (2 n eps sum|terms|), S assembled in long double."""
    nlc = W.shape[1]
    L = np.longdouble
    Wl, hpl = W.astype(L), hp.astype(L)
    S = Hd[:nlc, :nlc].astype(L) - Wl.T @ (Wl / hpl[:, None])
    mag = np.abs(Hd[:nlc, :nlc]).astype(L) + np.abs(Wl).T @ (np.abs(Wl) / hpl[:, None])
    tol = 2 * (W.shape[0] + 2) * np.finfo(np.float64).eps * mag
    err = np.abs(S_dev[:nlc, :nlc].astype(L) - S)
    return float(np.max(err / np.maximum(tol, np.finfo(np.float64).tiny), initial=0.0))


def backward_error(Hd, g, W, hp, gl, step):
    """eta = |A d + b|_inf / (|A|_inf |d|_inf + |b|_inf) on A = [[Hd, Wp^T], [Wp, diag(hp)]], b = [g; gl], in long double."""
    L = np.longdouble
    n, nlc = len(g), W.shape[1]
    Wp = np.zeros((len(hp), n), dtype=L); Wp[:, :nlc] = W
    dc, dl = step[:n].astype(L), step[n:].astype(L)
    Hl, hpl = Hd.astype(L), hp.astype(L)
    r = np.concatenate([Hl @ dc + Wp.T @ dl + g.astype(L), Wp @ dc + hpl * dl + gl.astype(L)])
    a_inf = max(np.max(np.abs(Hl).sum(axis=1) + np.abs(Wp).sum(axis=0)), np.max(np.abs(Wp).sum(axis=1) + np.abs(hpl), initial=0))
    b_inf = max(np.max(np.abs(g)), np.max(np.abs(gl), initial=0.0))
    dinf = float(np.max(np.abs(step)))
    return float(np.max(np.abs(r)) / (a_inf * L(dinf) + L(b_inf)))


def reference_step(Hd, g, W, hp, gl):
    """float64 numpy solve in the device's elimination order: landmark Schur complement, Cholesky, back substitution."""
    import scipy.linalg as sl
    n, nlc = len(g), W.shape[1]
    Wp = np.zeros((len(hp), n)); Wp[:, :nlc] = W
    S = Hd - Wp.T @ (Wp / hp[:, None])
    rhs = -(g - Wp.T @ (gl / hp))
    dc = sl.cho_solve(sl.cho_factor(S, lower=True), rhs)
    dl = -(gl + Wp @ dc) / hp
    return np.concatenate([dc, dl])


def condition(Hd, W, hp):
    n, nlc = Hd.shape[0], W.shape[1]
    Wp = np.zeros((len(hp), n)); Wp[:, :nlc] = W
    A = np.block([[Hd, Wp.T], [Wp, np.diag(hp)]])
    return float(np.linalg.cond(A, np.inf))


# ---------------------------------------------------------------------------------------------------------- CPU tests
# each rule as (label, field test) with the catalogue entries that must land on either side of it
RULES = {
    "fused ldw <= 72": (lambda p: p["ldw"] <= 72 and p["sb_elim"] and not p["n_leaf"], ["f11", "f11_td"], ["f12", "f11_stereo_ext"]),
    "k_schur_small": (lambda p: p["schur_small"] == 1, ["f15_td"], ["f16"]),
    "chol_smem after sb elimination": (lambda p: p["chol_smem"] == 1, ["f27"], ["f28"]),
    "sb_elim": (lambda p: p["sb_elim"] == 1, ["f32"], ["f33", "f12_imu_2_4"]),
    "k_chol ceiling": (lambda p: chol_global_smem_bytes(p["n_c"] + 1) <= SMEM_OPTIN - 16, ["f53"], ["f54"]),
    "leaf kept": (lambda p: p["n_leaf"] > 0, ["a2_f15", "a2_f16"], ["a2_f17", "a2_f15_two_remote_free"]),
    "hub_small": (lambda p: p["hub_small"] == 1, ["a2_f15"], ["a2_f16"]),
    "rec_stride 12": (lambda p: p["rec_stride"] == 12, ["f2_lm40", "f17", "f32"], ["f34", "anchor_const_f17"]),
    "gather_nosync": (lambda p: p["gather_nosync"] == 1, ["f11"], ["anchor_const_f17", "anchor_const_f33"]),
    "256-byte records": (lambda p: p["rec_stride"] == 32, ["stereo_td_f9", "stereo_td_f9_no1f2c", "stereo_td_f17_no1f2c", "stereo_td_f17", "f11_stereo_ext"], ["f11", "anchor_const_f34", "quad"]),
    "lm_mask width": (lambda p: p["n_lc"] // 32 < 64, ["a31_f11"], ["a32_f11"]),
}


def test_catalogue_hits_both_sides_of_every_rule():
    for label, (inside, below, above) in RULES.items():
        for name in below:
            assert inside(plan_of(name)), (label, name, plan_of(name))
        for name in above:
            assert not inside(plan_of(name)), (label, name, plan_of(name))
    # the neighbours of a boundary differ by one frame (or one parameter block)
    assert (plan_of("f11")["ldw"], plan_of("f11_td")["ldw"], plan_of("f12")["ldw"], plan_of("f11_stereo_ext")["ldw"]) == (72, 72, 80, 80)
    assert (plan_of("f15_td")["n_lc"], plan_of("f16")["n_lc"]) == (91, 96)
    f27, f28 = plan_of("f27"), plan_of("f28")
    assert f27["sb_elim"] and f28["sb_elim"] and chol_smem_bytes(f28["n_hub"] - 6) <= SMEM_OPTIN - 16 < chol_smem_bytes(f28["n_hub"])
    assert (plan_of("f32")["n_sbe"], plan_of("f33")["n_sbe"]) == (32, 33)
    assert chol_global_smem_bytes(plan_of("f53")["n_c"] + 1 + 15) > SMEM_OPTIN - 16            # 54 frames do not fit
    a16 = plan_of("a2_f16")
    assert a16["n_leaf"] == 1 and a16["hub0"] == 96 and not a16["hub_small"]                  # a 96-column leaf
    assert plan_of("a2_f17")["n_leaf"] == 0 and plan_of("a2_f17")["n_lc"] == 204
    assert plan_of("a2_f15_two_remote_free")["n_lc"] == 102                                    # 90 hub > 3/4 * 102
    assert (plan_of("a31_f11")["n_lc"], plan_of("a32_f11")["n_lc"]) == (2046, 2112)
    assert plan_of("a31_f11")["n_leaf"] == 30
    # the gathers' row buffers from a single tile to the widest window without leaves (f53: 10 tiles)
    assert plan_of("f2_lm1")["row_tiles"] == 1 and plan_of("f53")["row_tiles"] == 10


def test_catalogue_counts():
    """The record and tile counts the rules above rely on hold for the generated windows."""
    expect_records = {"f2_lm40": 1, "f17": 16, "f32": 31, "f34": 33, "anchor_const_f17": 16, "anchor_const_f18": 17,
                      "anchor_const_f33": 32, "anchor_const_f34": 33, "stereo_td_f9": 17, "stereo_td_f17": 33,
                      "stereo_td_f9_no1f2c": 16, "stereo_td_f17_no1f2c": 32}
    for name, k in expect_records.items():
        r = records_per_landmark(problem(name))
        assert r.min() == r.max() == k, (name, r.min(), r.max())
    assert records_per_landmark(problem("f33")).max() == 32 and plan_of("f33")["rec_stride"] == 12
    for n in (1, 31, 32, 33, 64, 65):
        pr = problem(f"f2_lm{n}")
        assert landmarks_per_pair(pr) == [n], (n, landmarks_per_pair(pr))
        assert plan_of(f"f2_lm{n}")["n_tile"] == (n + 31) // 32
        assert plan_of(f"f2_lm{n}")["n_g12"] == (n + 30) // 31
    assert plan_of("f17")["n_g12"] == 20                                                       # 2 landmarks of 16 records per chunk
    types = {name: set(np.unique(problem(name)["obs"]["type"]).tolist()) for name in ("depth", "quad", "f11_stereo_ext")}
    assert types["depth"] == {abi.PROJ_2F1C_DEPTH, abi.PROJ_DEPTH_PRIOR}
    assert {abi.PROJ_1F2C, abi.PROJ_2F2C} <= types["quad"] and {abi.PROJ_1F2C, abi.PROJ_2F2C} <= types["f11_stereo_ext"]
    # degenerate: constant frames 2 and 3 between free ones, a landmark only constant poses see, one record, an unobserved
    # free pose
    pr = problem("degenerate")
    assert pr["pose_const"].tolist() == [1, 0, 1, 1, 0, 0]
    o0 = pr["obs"][pr["obs"]["landmark_id"] == pr["lm_ids"][0]]
    assert len(o0) == 2 and all(pr["pose_const"][list(pr["frame_ids"]).index(f)] for f in np.concatenate([o0["frame_a"], o0["frame_b"]]))
    assert records_per_landmark(pr)[1] == 1
    assert pr["frame_ids"][5] not in set(pr["obs"]["frame_b"].tolist())
    for name in CATALOGUE:
        p = plan_of(name)
        assert p["n_c"] == p["n_lc"] + 9 * len(problem(name)["sb_ids"])


def _oracle(name):
    from oracle import orc
    pr = problem(name)
    o = orc.Oracle(); pr.load(o); o.debug_linearize()
    n = int(o.debug_get(abi.DBG_N_CAM, np.int64)[0]); nlc = int(o.debug_get(abi.DBG_N_LC, np.int64)[0])
    return o, n, nlc, len(pr["lm_ids"])


@pytest.mark.parametrize("name", ["f11", "f16", "a2_f15", "degenerate"])
def test_references_reproduce_the_oracle(name):
    """The Schur assembly and the eta criterion accept the oracle's own reduced system and GN step, and the reference
    solve in the device's elimination order agrees with the oracle's."""
    o, n, nlc, nl = _oracle(name)
    Hd, g, W, hp, gl = damped_views(o.debug_get, n, nlc, nl)
    assert nlc == plan_of(name)["n_lc"] and n == plan_of(name)["n_c"]
    assert schur_excess(o.debug_get(abi.DBG_S).reshape(n, n), Hd, W, hp) <= 1.0
    step = o.debug_get(abi.DBG_GN_STEP)
    ref = reference_step(Hd, g, W, hp, gl)
    eta_o, eta_r = backward_error(Hd, g, W, hp, gl, step), backward_error(Hd, g, W, hp, gl, ref)
    assert eta_r <= 1e-14 and eta_o <= max(ETA_FLOOR, 10 * eta_r), (eta_o, eta_r)
    assert relerr(ref, step) <= 1e-6


def test_criteria_are_sharp():
    """One landmark's contribution dropped from S, or a step perturbed by 1e-9 of its size, fails the criteria."""
    o, n, nlc, nl = _oracle("f16")
    Hd, g, W, hp, gl = damped_views(o.debug_get, n, nlc, nl)
    S = o.debug_get(abi.DBG_S).reshape(n, n)
    l = int(np.argmax(np.abs(W).sum(axis=1)))
    S_bad = S.copy(); S_bad[:nlc, :nlc] += np.outer(W[l], W[l]) / hp[l]
    assert schur_excess(S_bad, Hd, W, hp) > 1e3
    ref = reference_step(Hd, g, W, hp, gl)
    eta_r = backward_error(Hd, g, W, hp, gl, ref)
    bad = ref * (1 + 1e-9 * np.random.default_rng(0).standard_normal(len(ref)))
    assert backward_error(Hd, g, W, hp, gl, bad) > 100 * max(ETA_FLOOR, 10 * eta_r)


# ---------------------------------------------------------------------------------------------------------- GPU tests
def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _record(name, handle, **vals):
    """Appends the measured values to the JSON-lines file D2BA_ETA_LOG names (the DESIGN.md eta table)."""
    path = os.environ.get("D2BA_ETA_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(name=name, handle=handle, **vals)) + "\n")


def _check_window(s, w, name, handle, oracle_checks=True):
    """Plan-independent numerical checks of one window of a linearised handle; returns (GN step, eta)."""
    pr = problem(name)
    p = s.debug_plan(w)
    n, nlc, nl = p["n_c"], p["n_lc"], len(pr["lm_ids"])
    get = lambda item: s.debug_get(w, item)           # noqa: E731
    Hd, g, W, hp, gl = damped_views(get, n, nlc, nl)
    if oracle_checks:
        o, n_o, nlc_o, _ = _oracle(name)
        assert (n_o, nlc_o) == (n, nlc)
        for item in (abi.DBG_COST, abi.DBG_HCC, abi.DBG_GC, abi.DBG_HLL, abi.DBG_GL, abi.DBG_W):
            assert relerr(get(item), o.debug_get(item)) <= 1e-10, (name, item)
    ex = schur_excess(get(abi.DBG_S).reshape(n, n), Hd, W, hp)
    step = get(abi.DBG_GN_STEP)
    eta = backward_error(Hd, g, W, hp, gl, step)
    eta_ref = backward_error(Hd, g, W, hp, gl, reference_step(Hd, g, W, hp, gl))
    _record(name, handle, eta=eta, eta_ref=eta_ref, schur_excess=ex, plan=p)
    assert ex <= 1.0, (name, handle, ex)
    assert eta <= max(ETA_FLOOR, 10 * eta_ref), (name, handle, eta, eta_ref)
    return step, eta, (Hd, W, hp)


def _alone(name):
    from d2slam_b200.solver import Solver
    s = Solver(); problem(name).load(s, 0); s.finalize()
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_window_alone(name):
    s = _alone(name)
    plans, refusal = predict_handle([plan_of(name)], _n_sm())
    assert refusal == 0
    assert s.debug_plan(0) == plans[0], (name, s.debug_plan(0), plans[0])
    s.debug_linearize()
    _check_window(s, 0, name, "alone")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_window_fixed_schedule(name):
    """The first dogleg step, then 8 iterations on the device and in the oracle: same accepted steps, cost and state
    (test_gpu_parity's L3 bounds)."""
    from oracle import orc
    pr = problem(name)
    o = orc.Oracle(); pr.load(o)
    s = _alone(name)
    o.solve_fixed(1); s.solve_fixed(1)
    assert relerr(s.debug_get(0, abi.DBG_STEP), o.debug_get(abi.DBG_STEP)) <= 1e-6, name
    o = orc.Oracle(); pr.load(o)
    ro = o.solve_fixed(8)
    s = _alone(name)
    rs = s.solve_fixed(8)[0]
    assert ro.successful_steps == rs.successful_steps, name
    assert abs(rs.final_cost - ro.final_cost) <= 1e-7 * max(1.0, abs(ro.final_cost)), (name, rs.final_cost, ro.final_cost)
    d = state_diff(state_of(s, pr, 0), state_of(o, pr))
    assert d["pos"] <= 1e-6 and d["rot"] <= 1e-6, (name, d)


@pytest.mark.gpu
def test_mixed_handle():
    """The whole catalogue in one handle, padded with bench windows to 3 x SMs windows eligible for k_solve_small: the
    fused path, the 512-thread k_chol_smem and the widest row buffers apply at once.  Every window's normal equations
    equal the oracle's, its Schur complement and GN step pass the same checks as alone, and its GN step differs from the
    alone one by no more than the condition estimate allows."""
    from d2slam_b200.solver import Solver
    names = list(CATALOGUE)
    bench = synth.make_window(seed=4242, n_frames=11, n_landmarks=300)
    n_pad = 3 * _n_sm()
    s = Solver(max_windows=len(names) + n_pad)
    for i, name in enumerate(names):
        problem(name).load(s, i)
    for i in range(n_pad):
        bench.load(s, len(names) + i)
    s.finalize()
    plans, refusal = predict_handle([plan_of(n) for n in names] + [predict_plan(bench)] * n_pad, _n_sm())
    assert refusal == 0
    assert plans[0]["fused_solve"] == 1 and plans[0]["chol_threads"] == 512
    for i, name in enumerate(names):
        assert s.debug_plan(i) == plans[i], (name, s.debug_plan(i), plans[i])
    assert s.debug_plan(len(names)) == plans[len(names)]
    s.debug_linearize()
    for i, name in enumerate(names):
        step_m, eta_m, (Hd, W, hp) = _check_window(s, i, name, "mixed")
        a = _alone(name); a.debug_linearize()
        step_a, eta_a, _ = _check_window(a, 0, name, "alone", oracle_checks=False)
        kappa = condition(Hd, W, hp)
        diff = np.abs(step_m - step_a).max() / np.abs(step_a).max()
        _record(name, "mixed_vs_alone", diff=diff, kappa=kappa)
        assert diff <= 10 * kappa * (eta_m + eta_a + 1e-16), (name, diff, kappa, eta_m, eta_a)


@pytest.mark.gpu
def test_31_agent_window():
    """n_lc = 2046: the rhs column sits in the last of 64 landmark tiles, the widest window the masks describe."""
    name = "a31_f11"
    s = _alone(name)
    plans, refusal = predict_handle([plan_of(name)], _n_sm())
    assert refusal == 0 and s.debug_plan(0) == plans[0], (s.debug_plan(0), plans[0])
    s.debug_linearize()
    _check_window(s, 0, name, "alone", oracle_checks=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["f54", "a32_f11"])
def test_refusal_leaves_the_handle_usable(name):
    """A window beyond a limit is refused by d2ba_finalize with its code and the message of that limit (code 27 before
    any device work, code 23 when the kernel's shared-memory size is set, after the tile build was enqueued); after
    a reset the same handle solves a bench window."""
    from d2slam_b200.solver import D2BAError, Solver
    code = LARGE[name][1]
    assert predict_handle([plan_of(name)], _n_sm())[1] == code
    s = Solver()
    problem(name).load(s, 0)
    with pytest.raises(D2BAError, match=REFUSAL_MESSAGE[name]):
        s.finalize()
    s.reset()
    pr = synth.make_window(seed=4242, n_frames=11, n_landmarks=300)
    pr.load(s, 0); s.finalize()
    rep = s.solve_fixed(4)[0]
    assert rep.total_iterations == 4 and rep.final_cost < rep.initial_cost
