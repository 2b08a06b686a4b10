"""The sparse Cholesky's step at the front shapes where a multifrontal kernel goes wrong (include/d2pgo.h
d2pgo_set_linear_solver, d2slam_b200/csrc/d2pgo_chol.cu).  CPU: every graph family first proves, from the host analysis
(cholesky_symbolic) and the pattern of L that scipy factors under its permutation, that it produces the fronts it claims:
single fronts over 1 to 33 panels of 16 columns with every row residue mod the 8-row tensor-core tile, the largest front the
kernels take, update corners fed by several children, deep level chains, and degenerate structures.  GPU: each case's device
step, 4-DoF and 6-DoF at lambda 0, 1e-4, 1 and 1e4 on edges whose square-root information spans 1e-3 to 1e3, judged by its
backward error on the system the device factored against numpy's (test_pgo_cholesky.check_step); the bench graph against
scipy's sparse LU; bitwise reproducibility at the largest front."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from d2slam_b200 import pgo

import test_pgo_cholesky as tpc

LAMBDAS = (0.0, 1e-4, 1.0, 1e4)
# single fronts: a clique of n free poses, W = M = n D scalar columns; (n, panels of 16 columns) per block size
SINGLE = {6: [1, 3, 5, 40, 42, 43, 88], 4: [1, 4, 60, 63, 64, 68, 132]}
LARGEST = {6: 170, 4: 256}   # free poses of the largest clique the kernels take: 1020 and 1024 rows


# ------------------------------------------------------------------------------------------------ graph families
def _clique(nodes):
    nodes = np.asarray(nodes)
    a, b = np.triu_indices(len(nodes), 1)
    return nodes[a], nodes[b]


def _anchored(n_free, blocks):
    """pose 0 fixed and joined to every free pose 1..n_free, plus the given (ea, eb) blocks"""
    ea = np.concatenate([np.zeros(n_free, int)] + [a for a, _ in blocks])
    eb = np.concatenate([np.arange(1, n_free + 1)] + [b for _, b in blocks])
    fixed = np.zeros(n_free + 1, np.uint8); fixed[0] = 1
    return n_free + 1, fixed, ea, eb


def single(n):
    return _anchored(n, [_clique(np.arange(1, n + 1))])


def corners(k, c, s):
    """k cliques of c poses, each joined completely to a separator clique of s poses (numbered last)"""
    S = np.arange(1 + k * c, 1 + k * c + s)
    return _anchored(k * c + s, [_clique(np.r_[np.arange(1 + i * c, 1 + (i + 1) * c), S]) for i in range(k)])


def lattice(k):
    """a k x k grid with its horizontal, vertical and one diagonal neighbours; pose 0 fixed, joined to one corner"""
    idx = 1 + np.arange(k * k).reshape(k, k)
    ea = np.r_[0, idx[:, :-1].ravel(), idx[:-1, :].ravel(), idx[:-1, :-1].ravel()]
    eb = np.r_[1, idx[:, 1:].ravel(), idx[1:, :].ravel(), idx[1:, 1:].ravel()]
    fixed = np.zeros(k * k + 1, np.uint8); fixed[0] = 1
    return k * k + 1, fixed, ea, eb


def chain(n):
    fixed = np.zeros(n + 1, np.uint8); fixed[0] = 1
    return n + 1, fixed, np.arange(n), np.arange(1, n + 1)


def star(n):
    """n free poses, each joined to one of two fixed poses only: no free-free pair"""
    fixed = np.zeros(n + 2, np.uint8); fixed[:2] = 1
    return n + 2, fixed, np.r_[np.zeros(n, int), np.ones(n, int)], np.r_[np.arange(2, n + 2), np.arange(2, n + 2)]


def with_repeats(structure, repeat, selfs, seed=0):
    """the structure with `repeat` edges duplicated (half of them turned around) and `selfs` self loops on free poses"""
    n, fixed, ea, eb = structure
    rng = np.random.default_rng(seed)
    e = rng.choice(len(ea), repeat, replace=False)
    turn = rng.random(repeat) < 0.5
    loops = rng.choice(np.nonzero(fixed == 0)[0], selfs, replace=False)
    return n, fixed, np.r_[ea, np.where(turn, eb[e], ea[e]), loops], np.r_[eb, np.where(turn, ea[e], eb[e]), loops]


def isolated(structure, extra):
    """the structure and `extra` free poses no edge names"""
    n, fixed, ea, eb = structure
    return n + extra, np.r_[fixed, np.zeros(extra, np.uint8)], ea, eb


def two_components():
    """an anchored clique of 30 free poses and a clique of 20 free poses without a fixed one (its gauge is held by the damping
    alone, so it is solved at lambda > 0 only)"""
    n, fixed, ea, eb = single(30)
    a, b = _clique(np.arange(n, n + 20))
    return n + 20, np.r_[fixed, np.zeros(20, np.uint8)], np.r_[ea, a], np.r_[eb, b]


# name -> (structure, what it is about); every entry is checked by test_case_has_the_claimed_fronts for both block sizes
def cases():
    c = {}
    for D in (4, 6):
        for n in SINGLE[D]:
            c[f"single_{n}_{D}dof"] = (single(n), "single")
    c["largest_6dof"] = (single(LARGEST[6]), "single")
    c["largest_4dof"] = (single(LARGEST[4]), "single")
    c["corners_2_children"] = (corners(4, 10, 10), "corners")
    c["corners_3_children"] = (corners(5, 8, 12), "corners")
    c["lattice"] = (lattice(40), "lattice")
    c["chain"] = (chain(1000), "chain")
    c["no_free_pair"] = (star(40), "star")
    c["single_free_pose"] = (_anchored(1, []), "single")
    c["poses_without_edges"] = (isolated(single(20), 5), "isolated")
    c["repeats_and_self_loops_large_front"] = (with_repeats(single(120), 200, 40), "repeats")
    c["two_components"] = (two_components(), "components")
    return c


def case_dofs(name):
    if name.endswith("_6dof"):
        return (6,)
    if name.endswith("_4dof"):
        return (4,)
    return (4, 6)


# ------------------------------------------------------------------------------------------------ fronts from the pattern of L
def fronts(structure, D):
    """(analysis, [(W, M, children)] scalar per supernode) with M from the pattern of L: the free poses' block pattern under
    the analysis' permutation, factored by SuperLU in natural order (an M-matrix: no cancellation, the exact pattern)"""
    n, fixed, ea, eb = structure
    r = pgo.cholesky_symbolic(n, fixed, ea, eb, D)
    nf = r["free_poses"]
    pos = -np.ones(n, int); pos[r["perm"]] = np.arange(nf)
    keep = (pos[ea] >= 0) & (pos[eb] >= 0) & (ea != eb)
    a, b = pos[ea[keep]], pos[eb[keep]]
    B = sp.coo_matrix((np.ones(len(a)), (a, b)), shape=(nf, nf)).tocsr()
    B = ((B + B.T) > 0).astype(float)
    M_ = (sp.diags(np.asarray(B.sum(axis=1)).ravel() + 1.0) - B).tocsc()
    L = spla.splu(M_, permc_spec="NATURAL", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True)).L.tocsc()
    ptr, par = r["sn_ptr"], r["sn_parent"]
    nch = np.bincount(par[par >= 0], minlength=len(par))
    out = []
    for s in range(len(par)):
        f, l = ptr[s], ptr[s + 1]
        below = np.unique(L.indices[L.indptr[f]:L.indptr[l]])
        out.append(((l - f) * D, (l - f + int((below >= l).sum())) * D, int(nch[s])))
    return r, out


def levels(par):
    lv = np.zeros(len(par), int)
    for s in range(len(par)):   # parents come later
        if par[s] >= 0:
            lv[par[s]] = max(lv[par[s]], lv[s] + 1)
    return int(lv.max()) + 1 if len(par) else 0


@pytest.mark.parametrize("name", list(cases()))
def test_case_has_the_claimed_fronts(name):
    structure, kind = cases()[name]
    n, fixed, ea, eb = structure
    for D in case_dofs(name):
        r, fr = fronts(structure, D)
        W = np.array([f[0] for f in fr]); M = np.array([f[1] for f in fr]); ch = np.array([f[2] for f in fr])
        assert M.max(initial=0) == r["max_front_rows"] and W.max(initial=0) == r["max_front_cols"], (name, D)
        assert levels(r["sn_parent"]) == r["levels"], (name, D)
        assert np.all(M >= W)
        nfree = int((fixed == 0).sum())
        if kind == "single":
            assert len(fr) == 1 and W[0] == M[0] == nfree * D, (name, D, fr)
        elif kind == "corners":   # a front fed by several children, each with an update corner
            s = int(np.argmax(ch))
            kids = np.nonzero(r["sn_parent"] == s)[0]
            assert ch[s] >= (3 if "3" in name else 2) and np.all(M[kids] > W[kids]), (name, D, fr)
        elif kind == "lattice":   # fronts of several hundred rows with update corners, fed by several children
            assert 300 <= r["max_front_rows"] <= 1024 and np.any((M > W) & (M >= 300)) and ch.max() >= 3, (name, D, r)
            assert r["levels"] >= 8
        elif kind == "chain":     # a deep tree: many levels of small fronts
            assert r["levels"] >= 20 and r["levels_fundamental"] >= 50, (name, D, r)
        elif kind == "star":
            assert r["block_pairs"] == 0 and len(fr) == nfree and np.all(M == D) and r["levels"] == 1
        elif kind == "isolated":
            roots = np.nonzero(r["sn_parent"] == -1)[0]
            assert sum(1 for s in roots if ch[s] == 0 and M[s] == D) >= 5, (name, D, fr)
        elif kind == "repeats":
            free = fixed == 0
            pairs = {(min(a, b), max(a, b)) for a, b in zip(ea, eb) if a != b and free[a] and free[b]}
            assert r["block_pairs"] == len(pairs) < int((free[ea] & free[eb] & (ea != eb)).sum())
            assert np.any(ea == eb) and r["max_front_rows"] >= 480
        elif kind == "components":
            assert int((r["sn_parent"] == -1).sum()) >= 2
        assert r["max_front_rows"] <= 1024
    if name.startswith("largest"):   # one pose more is refused by the analysis' front limit
        D = case_dofs(name)[0]
        assert pgo.cholesky_symbolic(*single(LARGEST[D] + 1), D)["max_front_rows"] > 1024


def test_single_fronts_cover_every_panel_and_tile_residue():
    for D in (4, 6):
        W = np.array(SINGLE[D]) * D
        panels = -(-W // 16)
        assert {1, 15, 16, 17, 33} <= set(panels.tolist()), (D, panels)
        assert set((W % 8).tolist()) == ({0, 4} if D == 4 else {0, 2, 4, 6}), (D, W % 8)
        assert len(set((W % 16).tolist())) >= (3 if D == 4 else 5)
    assert LARGEST[6] * 6 == 1020 and LARGEST[4] * 4 == 1024


# ------------------------------------------------------------------------------------------------ GPU
def graph(structure, D, seed=0, scale=(-3.0, 3.0)):
    """poses and measurements for a structure: random true poses, measurements of the true relative poses with noise, the
    initial guess off the truth (so g != 0), square-root information s (I + 0.3 U) with s log-uniform over 10^scale and U a
    random strictly upper triangle"""
    n, fixed, ea, eb = structure
    rng = np.random.default_rng(seed)
    E = len(ea)
    S = np.eye(D) + 0.3 * np.triu(rng.normal(size=(E, D, D)), 1)
    S *= (10.0 ** rng.uniform(*scale, E))[:, None, None]
    if D == 6:
        gt = np.zeros((n, 7)); gt[:, :3] = rng.uniform(-5, 5, (n, 3)); gt[:, 3:] = pgo._qexp(rng.normal(0, 0.5, (n, 3)))
        rel = pgo.relative_pose(gt[ea], gt[eb])
        rel[:, :3] += rng.normal(0, 0.05, (E, 3))
        q = pgo._qmul(rel[:, 3:7], pgo._qexp(rng.normal(0, 0.02, (E, 3)))); rel[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
        init = gt.copy(); init[:, :3] += rng.normal(0, 0.1, (n, 3))
        q = pgo._qmul(init[:, 3:7], pgo._qexp(rng.normal(0, 0.05, (n, 3)))); init[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    else:
        gt = np.c_[rng.uniform(-5, 5, (n, 3)), rng.uniform(-3, 3, n)]
        c, s_ = np.cos(-gt[ea, 3]), np.sin(-gt[ea, 3]); v = gt[eb, :3] - gt[ea, :3]
        rel = np.c_[c * v[:, 0] - s_ * v[:, 1], s_ * v[:, 0] + c * v[:, 1], v[:, 2], pgo.normalize_angle(gt[eb, 3] - gt[ea, 3])]
        rel += rng.normal(0, 0.05, (E, 4)) * np.array([1, 1, 1, 0.4])
        rel[:, 3] = pgo.normalize_angle(rel[:, 3])
        init = gt + rng.normal(0, 0.1, (n, 4)) * np.array([1, 1, 1, 0.5]); init[:, 3] = pgo.normalize_angle(init[:, 3])
    init[fixed != 0] = gt[fixed != 0]
    ids = np.arange(n, dtype=np.int64) * 7 + 3
    return dict(ids=ids, init=init, fixed=fixed, ea=ea, eb=eb, id_a=ids[ea], id_b=ids[eb], rel=rel, sqrt_info=S.reshape(E, D * D))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(cases()))
def test_step_is_backward_stable(name):
    structure, kind = cases()[name]
    for D in case_dofs(name):
        g = graph(structure, D, seed=len(name) + D)
        s = tpc.device(g, D)
        st = s.cholesky_stats()
        assert st["max_front_rows"] <= 1024
        for lam in LAMBDAS:
            if kind == "components" and lam == 0.0:
                continue
            tpc.check_step(s, g, D, lam, label=name)
        if name.startswith("largest"):
            assert st["max_front_rows"] == LARGEST[D] * D
        s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 6])
def test_one_pose_more_than_the_largest_front_is_refused(D):
    g = graph(single(LARGEST[D] + 1), D)
    s = tpc.device(g, D)
    with pytest.raises(RuntimeError, match="front of"):
        s.debug_exact_step(1e-4)
    assert s.cholesky_stats()["factorizations"] == 0
    s.close()


@pytest.mark.gpu
def test_largest_front_steps_are_bitwise_reproducible():
    for D in (4, 6):
        g = graph(single(LARGEST[D]), D, seed=5)
        out = []
        for _ in range(2):
            s = tpc.device(g, D)
            out.append([s.debug_exact_step(lam) for lam in LAMBDAS])
            s.close()
        assert all(np.array_equal(a, b) for a, b in zip(*out)), D


def bench_cases():
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    return {"6dof": (g, 6, None), "4dof": (pgo.pose_graph_to_4d(g, seed=7), 4, None),
            "6dof_gravity": (g, 6, pgo.make_gravity_case(g, seed=7)["ego"])}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof", "4dof", "6dof_gravity"])
def test_bench_graph_step_against_sparse_lu(name):
    """the bench graph (9 999 free poses): the device system against the records' sums entry by entry, eta of the device
    step and of scipy's sparse LU of the same system, and their forward difference within a 1-norm condition estimate"""
    g, D, ego = bench_cases()[name]
    s = tpc.device(g, D, ego)
    lam = 1e-4
    dx = s.debug_exact_step(lam)
    fx = np.asarray(g["fixed"]) != 0
    A, b = tpc.device_system(s, g, D)
    _, _, ulps = tpc.check_assembly(s, g, D, lam, A, b, with_priors=ego is not None)
    assert s.cholesky_stats()["max_front_rows"] == 70 * D   # 420 x 384 in 6-DoF
    x = dx[~fx].ravel()
    lu = spla.splu(A.tocsc(), permc_spec="MMD_AT_PLUS_A")
    ref = lu.solve(b)
    e, e_ref = tpc.eta(A, x, b), tpc.eta(A, ref, b)
    inv = spla.LinearOperator(A.shape, matvec=lu.solve, rmatvec=lambda v: lu.solve(v, trans="T"), dtype=float)
    cond = spla.onenormest(A) * spla.onenormest(inv)
    fwd = np.abs(x - ref).max() / np.abs(ref).max()
    print(f"bench {name} lambda {lam:g}: n {A.shape[0]}, eta device {e:.2e} scipy LU {e_ref:.2e}, cond1 ~ {cond:.1e}, "
          f"forward diff {fwd:.1e}, assembly {ulps:.1f} eps x magnitudes")
    assert e <= max(tpc.ETA_BOUND, 10 * e_ref), (name, e, e_ref)
    assert fwd <= 10 * cond * (e + e_ref), (name, fwd, cond)
    s.close()
