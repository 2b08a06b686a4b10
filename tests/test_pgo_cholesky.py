"""Pose graph with exact LM steps from the sparse Cholesky (include/d2pgo.h d2pgo_set_linear_solver, d2pgo's
SPARSE_NORMAL_CHOLESKY).  CPU: the host symbolic analysis (a permutation of the free poses, nnz(L) against scipy's factor of
the permuted pattern, a supernodal tree, determinism) on graphs with repeated pairs, self loops, fixed ends, two components and
a pose without edges; the LM oracle against the sparse-direct Gauss-Newton oracles.  GPU: the device step's backward error on
the system it factored against numpy's, that system against the parity hooks' records entry by entry (plain, with gravity
priors and with ARock proximal terms), LM parity with the oracle iteration by iteration, the converged solution with
default settings, ARock with Cholesky local solves, reproducibility, switching back to PCG, refusals and failed pivots."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from d2slam_b200 import pgo, synth
from oracle import pgo4d_oracle as p4
from oracle import pgo_arock_oracle as ao
from oracle import pgo_gravity_oracle as go
from oracle import pgo_lm_oracle as lo
from oracle import pgo_oracle as po

import test_pgo_arock as tpa


def small_graph(seed=3, n_agents=3, n=60, loops=150):
    return pgo.make_pose_graph(seed=seed, n_agents=n_agents, poses_per_agent=n, loops=loops)


def with_extras(g, repeat=6, selfs=4, seed=0):
    """g with `repeat` edges duplicated (same pair, same measurement turned around or not) and `selfs` self loops."""
    rng = np.random.default_rng(seed)
    ea, eb, rel, si = list(g["ea"]), list(g["eb"]), list(g["rel"]), list(g["sqrt_info"])
    E = len(g["ea"])
    for e in rng.choice(E, repeat, replace=False):
        if rng.random() < 0.5:
            ea.append(g["ea"][e]); eb.append(g["eb"][e]); rel.append(g["rel"][e])
        else:
            ea.append(g["eb"][e]); eb.append(g["ea"][e]); rel.append(_inverse(g["rel"][e]))
        si.append(g["sqrt_info"][e])
    N = len(g["ids"])
    for i in rng.choice(np.arange(1, N), selfs, replace=False):
        ea.append(i); eb.append(i)
        r = np.zeros(len(g["rel"][0])); r[:3] = rng.normal(0, 0.05, 3)
        if len(r) == 7:
            r[3:7] = pgo._qexp(rng.normal(0, 0.02, 3))
        else:
            r[3] = rng.normal(0, 0.02)
        rel.append(r); si.append(g["sqrt_info"][0])
    ea = np.array(ea); eb = np.array(eb)
    ids = np.asarray(g["ids"])
    return dict(g, ea=ea, eb=eb, id_a=ids[ea], id_b=ids[eb], rel=np.array(rel), sqrt_info=np.array(si))


def pose_diff6(a, b):
    """largest position difference and largest attitude difference 2 |q_a - q_b| (sign-aligned), which resolves angles far
    below the arccos-based pose_errors"""
    qa, qb = a[:, 3:7], b[:, 3:7]
    sgn = np.where((qa * qb).sum(axis=1) < 0, -1.0, 1.0)[:, None]
    return float(np.linalg.norm(a[:, :3] - b[:, :3], axis=1).max()), float(2 * np.linalg.norm(qa - sgn * qb, axis=1).max())


def _inverse(r):
    """the measurement of an edge turned around: 6-DoF T^-1; 4-DoF [-Rz(-dyaw) p, N(-dyaw)]"""
    if len(r) == 4:
        c, s_ = np.cos(-r[3]), np.sin(-r[3])
        return np.array([-(c * r[0] - s_ * r[1]), -(s_ * r[0] + c * r[1]), -r[2], pgo.normalize_angle(-r[3])])
    qi = pgo._qconj(r[3:7])
    return np.concatenate([-pgo._qrot(qi, r[:3]), qi])


# ------------------------------------------------------------------------------------------------ CPU: symbolic analysis
def symbolic_cases():
    g = small_graph()
    N = len(g["ids"]); fx = np.asarray(g["fixed"])
    cases = {"bench_like": (N, fx, g["ea"], g["eb"])}
    x = with_extras(g)
    cases["repeated_pairs_and_self_loops"] = (N, fx, x["ea"], x["eb"])
    f2 = fx.copy(); f2[[0, 60, 61, 130]] = 1
    cases["fixed_ends"] = (N, f2, g["ea"], g["eb"])
    h = small_graph(seed=5, n_agents=1, n=80, loops=40)
    n1 = len(h["ids"])
    cases["two_components"] = (2 * n1, np.r_[h["fixed"], h["fixed"]], np.r_[h["ea"], h["ea"] + n1], np.r_[h["eb"], h["eb"] + n1])
    cases["pose_without_edges"] = (N + 3, np.r_[fx, np.zeros(3, np.uint8)], g["ea"], g["eb"])
    return cases


def scipy_nnz(n, fixed, ea, eb, perm):
    """nonzeros of L of the block pattern (free poses, permuted by perm) with random SPD values, by SuperLU in natural order"""
    free = np.nonzero(np.asarray(fixed) == 0)[0]
    pos = -np.ones(n, int); pos[perm] = np.arange(len(perm))
    keep = (pos[ea] >= 0) & (pos[eb] >= 0) & (ea != eb)
    a, b = pos[ea[keep]], pos[eb[keep]]
    rng = np.random.default_rng(1)
    A = sp.coo_matrix((rng.uniform(0.1, 1.0, len(a)), (a, b)), shape=(len(free), len(free))).tocsr()
    A = A + A.T
    M = (sp.diags(np.asarray(abs(A).sum(axis=1)).ravel() + 1.0) - A).tocsc()
    return spla.splu(M, permc_spec="NATURAL", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True)).L.nnz


@pytest.mark.parametrize("name", list(symbolic_cases()))
def test_symbolic_analysis(name):
    n, fixed, ea, eb = symbolic_cases()[name]
    r = pgo.cholesky_symbolic(n, fixed, ea, eb, 6)
    free = np.nonzero(np.asarray(fixed) == 0)[0]
    assert r["free_poses"] == len(free)
    assert sorted(r["perm"].tolist()) == free.tolist()                       # a permutation of the free poses
    assert r["nnz_L"] == scipy_nnz(n, fixed, np.asarray(ea), np.asarray(eb), r["perm"])
    assert r["nnz_L_stored"] >= r["nnz_L"]
    S = r["supernodes"]
    ptr, par = r["sn_ptr"], r["sn_parent"]
    assert ptr[0] == 0 and ptr[-1] == len(free) and np.all(np.diff(ptr) > 0)
    assert np.all((par == -1) | (par > np.arange(S)))                        # parents come later: a forest
    roots = int((par == -1).sum())
    assert roots >= 1 and (name != "two_components" or roots >= 2)
    assert r["levels"] <= r["levels_fundamental"] and r["supernodes"] <= r["supernodes_fundamental"]
    r2 = pgo.cholesky_symbolic(n, fixed, ea, eb, 6)
    for k in r:
        assert np.array_equal(np.asarray(r[k]), np.asarray(r2[k])), k


def test_symbolic_pair_count_and_refusals():
    g = small_graph()
    x = with_extras(g)
    N = len(g["ids"]); free = g["fixed"] == 0
    keep = free[x["ea"]] & free[x["eb"]] & (x["ea"] != x["eb"])
    pairs = {(min(a, b), max(a, b)) for a, b in zip(x["ea"][keep], x["eb"][keep])}
    assert pgo.cholesky_symbolic(N, g["fixed"], x["ea"], x["eb"], 4)["block_pairs"] == len(pairs)
    with pytest.raises(RuntimeError):
        pgo.cholesky_symbolic(N, g["fixed"], x["ea"], x["eb"], 5)
    with pytest.raises(RuntimeError):
        pgo.cholesky_symbolic(N, g["fixed"], np.r_[x["ea"], N], np.r_[x["eb"], 0], 6)


def test_symbolic_bench_graph_counts():
    g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    r = pgo.cholesky_symbolic(len(g["ids"]), g["fixed"], g["ea"], g["eb"], 6)
    assert r["free_poses"] == 9999 and r["block_pairs"] == 26634
    assert r["max_front_rows"] <= 1024
    print({k: v for k, v in r.items() if not isinstance(v, np.ndarray)})


# ------------------------------------------------------------------------------------------------ CPU: the LM oracle
def problem6(g, priors=False, selfs=False):
    x = with_extras(g) if selfs else g
    if not priors:
        return lo.Problem(x["init"], x["fixed"], x["ea"], x["eb"], x["rel"], x["sqrt_info"]), x, None
    c = pgo.make_gravity_case(x, seed=2)
    n = len(x["ids"])
    pri = (np.arange(n), go.ego_gravity(c["ego"]), np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (n, 1, 1)))
    return lo.Problem(x["init"], x["fixed"], x["ea"], x["eb"], x["rel"], x["sqrt_info"], *pri), x, c["ego"]


def problem4(seed=1):
    h = pgo.pose_graph_to_4d(small_graph(seed=seed, n=40, loops=100), seed=seed + 100)
    return lo.Problem(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"]), h


def test_lm_oracle_reaches_the_gauss_newton_optimum():
    prob, g, _ = problem6(small_graph(n=40, loops=100))
    x, hist, rep = lo.lm_solve(prob, max_iterations=100, lambda0=1e-6, function_tolerance=1e-15)
    y, _ = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=60, ftol=1e-15)
    dp, dr = pose_diff6(x, y)
    assert dp < 1e-8 and dr < 1e-8, (dp, dr)
    prob4, h = problem4()
    x4, _, _ = lo.lm_solve(prob4, max_iterations=100, lambda0=1e-6, function_tolerance=1e-15)
    y4, _ = p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"], iters=60, ftol=1e-15)
    assert np.abs(x4[:, :3] - y4[:, :3]).max() < 1e-8 and np.abs(pgo.normalize_angle(x4[:, 3] - y4[:, 3])).max() < 1e-8


# ------------------------------------------------------------------------------------------------ GPU
def device(g, dof=6, ego=None, linear_solver="sparse_cholesky", **kw):
    s = pgo.PgoSolver(pose_dof=dof, linear_solver=linear_solver, **kw)
    if dof == 4:
        s.set_poses_4d(g["ids"], g["init"], g["fixed"]); s.add_edges_4d(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    else:
        s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
        if ego is not None:
            s.add_gravity_priors(g["ids"], ego)
    return s


# ------------------------------------------------------------------------------------------------ the step's backward error
# A device step dx is judged by its normwise backward error on the system the device factored, read back through
# debug_cholesky_system:  eta = |A dx - b|_inf / (|A|_inf |dx|_inf + |b|_inf), the residual evaluated exactly enough (long
# double) that eta measures the solver alone.  A backward-stable Cholesky leaves eta at a small multiple of the unit roundoff
# whatever the conditioning; an indexing or assembly slip in the factor or the solves leaves far more.  That the device
# assembled the right system is checked separately and componentwise: each entry of its A and b against the same sums formed
# here from the edge, prior and proximal-term records, within a multiple of eps times the sums of magnitudes (any summation
# order stays inside that; a wrong or missing term does not).
# Measured on an H100 80GB HBM3 (700 W limit) over every case here and in test_pgo_cholesky_shapes.py: device eta 2e-18 to
# 4.6e-16 (the largest at the 1024-row front), the reference solves' 4e-18 to 2e-16, the device at most 6.4 times the
# reference's; assembly differences at most 16 eps times the magnitudes (the 170-pose clique), 5 at the bench graph.
ETA_BOUND = 2e-15          # the device's eta stays below max(ETA_BOUND, 10 eta of the reference solve of the same system)
ASSEMBLY_ULPS = 2          # |A_dev - A| <= ASSEMBLY_ULPS * n * eps * (sums of magnitudes), n = k D + 2 products per entry at most


def _block_coo(pa, pb, B, D):
    """COO triplets of the D x D blocks B[k] at block (pa[k], pb[k])"""
    ar = np.arange(D)
    rows = np.broadcast_to(np.asarray(pa)[:, None, None] * D + ar[None, :, None], B.shape)
    cols = np.broadcast_to(np.asarray(pb)[:, None, None] * D + ar[None, None, :], B.shape)
    return rows.ravel(), cols.ravel(), B.ravel()


def _coo_csr(trip, n):
    rows, cols, vals = (np.concatenate(v) for v in zip(*trip))
    return sp.coo_matrix((vals, (rows, cols)), shape=(n, n)).tocsr()


def records(s, g, dof, with_priors=False, arock_poses=None):
    """The handle's own edge, gravity-prior (one per pose) and (arock_poses: the pose of each dual in table order)
    proximal-term records at the current poses, as factor groups (poses of each Jacobian slot, r [R, m], Jacobians [R, m, D]
    per slot)"""
    D = dof; N = len(g["ids"])
    rec = s.debug_edges()
    factors = [((np.asarray(g["ea"]), np.asarray(g["eb"])), rec[:, :D],
                (rec[:, D:D + D * D].reshape(-1, D, D), rec[:, D + D * D:].reshape(-1, D, D)))]
    if with_priors:
        pr = s.debug_gravity_priors()
        factors.append(((np.arange(N),), pr[:, :3], (pr[:, 3:].reshape(-1, 3, 6),)))
    if arock_poses is not None:
        tr = s.debug_arock_terms(len(arock_poses))
        factors.append(((np.asarray(arock_poses),), tr[:, :D], (tr[:, D:].reshape(-1, D, D),)))
    return factors


def assemble(s, g, dof, lam, with_priors=False, arock_poses=None, magnitude=False, factors=None):
    """(A, b, terms) of (J^T J + diag(lam d + 1e-12)) dx = -J^T r over the free poses (D rows per free pose, in pose order;
    A scipy CSR) from the records (factors, or the handle's own: records()); terms = the largest number of records touching
    one pose.  magnitude: the same sums over |J| and |r| (b then holds +sum |J|^T |r|)."""
    D = dof; N = len(g["fixed"])
    f = np.abs if magnitude else (lambda v: v)
    factors = records(s, g, dof, with_priors, arock_poses) if factors is None else factors
    trip, gv, d, count = [], np.zeros(N * D), np.zeros(N * D), np.zeros(N, int)
    for poses, r, Js in factors:
        r, Js = f(r), tuple(f(J) for J in Js)
        for pa, Ja in zip(poses, Js):
            idx = (pa[:, None] * D + np.arange(D)).ravel()
            gv += np.bincount(idx, np.einsum("eka,ek->ea", Ja, r).ravel(), N * D)
            d += np.bincount(idx, (Ja ** 2).sum(axis=1).ravel(), N * D)
            count += np.bincount(pa, minlength=N)
            for pb, Jb in zip(poses, Js):
                trip.append(_block_coo(pa, pb, np.einsum("eka,ekb->eab", Ja, Jb), D))
    free = np.repeat(np.asarray(g["fixed"]) == 0, D)
    A = _coo_csr(trip, N * D)[free][:, free] + sp.diags(lam * d[free] + 1e-12)
    return A.tocsr(), (gv if magnitude else -gv)[free], int(count.max())


def device_system(s, g, dof):
    """(A, b) the device factored in its last step (debug_cholesky_system), in assemble's layout"""
    D = dof; N = len(g["ids"])
    m = s.debug_cholesky_system()
    fx = np.asarray(g["fixed"]) != 0
    assert np.all(m["diag"][fx] == 0.0) and np.all(m["b"][fx] == 0.0)
    fi = np.nonzero(~fx)[0]
    col = -np.ones(N, int); col[fi] = np.arange(len(fi))
    a, b = col[m["pairs"][:, 0]], col[m["pairs"][:, 1]]
    assert np.all(a >= 0) and np.all(b >= 0) and np.all(m["pairs"][:, 0] < m["pairs"][:, 1])
    trip = [_block_coo(np.arange(len(fi)), np.arange(len(fi)), m["diag"][fi], D),
            _block_coo(a, b, m["pair_blocks"], D), _block_coo(b, a, m["pair_blocks"].transpose(0, 2, 1), D)]
    return _coo_csr(trip, len(fi) * D), m["b"][fi].ravel()


def residual(A, x, b):
    """|A x - b|_inf with every product and sum in long double"""
    assert np.finfo(np.longdouble).eps < 1e-18
    A = A.tocsr(); ld = np.longdouble
    prod = A.data.astype(ld) * x.astype(ld)[A.indices]
    Ax = np.zeros(A.shape[0], ld)
    nz = np.diff(A.indptr) > 0
    Ax[nz] = np.add.reduceat(prod, A.indptr[:-1][nz]) if prod.size else 0
    return float(np.abs(Ax - b.astype(ld)).max()) if len(b) else 0.0


def eta(A, x, b):
    """normwise backward error of x in A x = b"""
    den = float(abs(A).sum(axis=1).max()) * float(np.abs(x).max(initial=0.0)) + float(np.abs(b).max(initial=0.0))
    res = residual(A, x, b)
    return res / den if den > 0 else res


def check_assembly(s, g, dof, lam, A, b, with_priors=False, arock_poses=None):
    """the device's A and b entry by entry against the records' sums; returns the largest |difference| / its allowance"""
    A0, b0, k = assemble(s, g, dof, lam, with_priors, arock_poses)
    Am, bm, _ = assemble(s, g, dof, lam, with_priors, arock_poses, magnitude=True)
    tol = ASSEMBLY_ULPS * (k * dof + 2) * np.finfo(float).eps
    over_A = (abs(A - A0) - tol * Am).tocsr()
    over_b = np.abs(b - b0) - tol * bm
    assert over_A.nnz == 0 or over_A.data.max() <= 0.0, ("A", over_A.data.max())
    assert over_b.max(initial=-1.0) <= 0.0, ("b", over_b.max())
    eps = np.finfo(float).eps
    w = abs(A - A0).tocoo()
    dA = (w.data / np.maximum(np.asarray(Am.tocsr()[w.row, w.col]).ravel() * eps, 1e-300)).max() if w.nnz else 0.0
    db = (np.abs(b - b0) / np.maximum(bm * eps, 1e-300)).max(initial=0.0)
    return A0, b0, float(max(dA, db))


def check_step(s, g, dof, lam, with_priors=False, arock_poses=None, label=""):
    """one device step at lam judged by eta on the system it factored (assembly checked first) against numpy's solve of
    that system; returns (eta device, eta numpy)"""
    dx = s.debug_exact_step(lam)
    fx = np.asarray(g["fixed"]) != 0
    assert np.all(dx[fx] == 0.0)
    A, b = device_system(s, g, dof)
    _, _, ulps = check_assembly(s, g, dof, lam, A, b, with_priors, arock_poses)
    x = dx[~fx].ravel()
    n = A.shape[0]
    ref = x if n == 0 else np.linalg.solve(A.toarray(), b) if n <= 3000 else spla.splu(A.tocsc(), permc_spec="MMD_AT_PLUS_A").solve(b)
    e, e_ref = eta(A, x, b), eta(A, ref, b)
    print(f"{label} {dof}-DoF lambda {lam:g}: n {A.shape[0]}, eta device {e:.2e} reference {e_ref:.2e}, assembly {ulps:.1f} eps x magnitudes")
    assert e <= max(ETA_BOUND, 10 * e_ref), (label, dof, lam, e, e_ref)
    return e, e_ref


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["6dof", "6dof_gravity", "4dof"])
def test_exact_step_equals_the_dense_solve(case):
    g = with_extras(small_graph(n=30, loops=80), repeat=8, selfs=4)
    g["fixed"] = g["fixed"].copy(); g["fixed"][[0, 45]] = 1          # edges to fixed poses at both ends
    dof, ego = 6, None
    if case == "4dof":
        h = pgo.pose_graph_to_4d(small_graph(n=30, loops=80), seed=9)
        g = with_extras(h, repeat=8, selfs=4)
        g["fixed"] = g["fixed"].copy(); g["fixed"][[0, 45]] = 1
        dof = 4
    if case == "6dof_gravity":
        ego = pgo.make_gravity_case(g, seed=3)["ego"]
    s = device(g, dof, ego)
    for lam in (0.0, 1e-4, 1.0, 1e4):
        check_step(s, g, dof, lam, ego is not None, label=case)
    assert s.cholesky_stats()["free_poses"] == int((g["fixed"] == 0).sum())
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
def test_exact_step_with_arock_proximal_terms_equals_the_dense_solve(dof):
    """agent 0 of a 3-agent ARock run after one round, whose local problem is converged, so g is a sum of terms that cancel
    to ~1e-8 of their size: the device system against the records' sums componentwise, and eta on the device system.  Also
    shows why a residual relative to |g| in the records' own float64 sums cannot judge the step here: two summation orders
    of g differ by eps times the terms, which is 1e-9 to 1e-8 of |g| itself."""
    gg = tpa.graph(dof)
    agents = tpa.device_agents(gg, tpa.SHIPPED["default"], solver_kw=dict(linear_solver="sparse_cholesky"))
    pgo.arock_run(agents, 1)
    a = agents[0]
    sp_ = a.split
    assert sp_["fixed"].sum() == 1
    pos = {int(i): k for k, i in enumerate(sp_["ids"])}
    g = dict(ids=sp_["ids"], fixed=sp_["fixed"], ea=np.array([pos[int(i)] for i in sp_["id_a"]]), eb=np.array([pos[int(i)] for i in sp_["id_b"]]))
    duals = sorted(a.duals())
    assert duals
    arock_poses = [pos[f] for _, f in duals]
    for lam in (0.0, 1e-4, 1.0, 1e4):
        check_step(a.s, g, dof, lam, arock_poses=arock_poses, label="arock")
        A, b = device_system(a.s, g, dof)
        _, b0, _ = assemble(a.s, g, dof, lam, arock_poses=arock_poses)
        _, bm, _ = assemble(a.s, g, dof, lam, arock_poses=arock_poses, magnitude=True)
        print(f"arock {dof}-DoF lambda {lam:g}: |b| / sum |J^T r| = {np.abs(b).max() / bm.max():.1e}, "
              f"|b_device - b_records| / |b| = {np.abs(b - b0).max() / np.abs(b).max():.1e}")
    for x in agents:
        x.close()


def device_history(g, dof, ego, iters, **kw):
    """(final cost, accepted) after k = 1..iters LM iterations, each from the initial poses"""
    out = []
    for k in range(1, iters + 1):
        s = device(g, dof, ego, max_iterations=k, **kw)
        r = s.solve()
        out.append((r.final_cost, r.accepted, r.iterations, r.converged))
        x = s.get_poses_4d(g["ids"]) if dof == 4 else s.get_poses(g["ids"])
        s.close()
        if r.iterations < k:
            break
    return out, x


def lm_cases():
    g6 = small_graph(seed=11, n=40, loops=100)
    h4 = pgo.pose_graph_to_4d(small_graph(seed=12, n=40, loops=100), seed=12)
    return {"6dof": (g6, 6, False), "4dof": (h4, 4, False), "6dof_gravity": (small_graph(seed=13, n=40, loops=100), 6, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof", "4dof", "6dof_gravity"])
def test_lm_iterations_match_the_oracle(name):
    g, dof, grav = lm_cases()[name]
    if dof == 4:
        yaw = g["init"][:, 3]
        assert np.abs(yaw).max() < np.pi - 0.05, "the parity case keeps its yaws away from +-pi"
        prob = lo.Problem(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"]); ego = None
    else:
        prob, g, ego = problem6(g, priors=grav)
    cfg = dict(lambda0=1e-4, function_tolerance=1e-12)
    x_o, hist, rep = lo.lm_solve(prob, max_iterations=12, **cfg)
    dev, x_d = device_history(g, dof, ego, len(hist), **cfg)
    acc = 0
    for k, (cand, ok) in enumerate(hist):
        acc += ok
        cost_d, acc_d = dev[k][0], dev[k][1]
        assert acc_d == acc, (k, acc_d, acc)
        want = cand if ok else (dev[k - 1][0] if k else rep["initial_cost"])
        if ok:
            assert abs(cost_d - want) <= 1e-9 * abs(want), (k, cost_d, want)
    if dof == 4:
        assert np.abs(x_d[:, :3] - x_o[:, :3]).max() < 1e-8 and np.abs(pgo.normalize_angle(x_d[:, 3] - x_o[:, 3])).max() < 1e-8
    else:
        dp, dr = pose_diff6(x_d, x_o)
        assert dp < 1e-8 and dr < 1e-8, (dp, dr)


@pytest.mark.gpu
def test_default_settings_reach_the_sparse_direct_optimum():
    g = small_graph(seed=21, n=60, loops=150)
    s = device(g, 6)
    r = s.solve()
    x = s.get_poses(g["ids"])
    assert r.pcg_iterations == 0 and r.final_cost < r.initial_cost
    y, _ = po.solve(g["init"], g["fixed"], g["ea"], g["eb"], g["rel"], g["sqrt_info"], iters=60, ftol=1e-15)
    dp, dr = pose_diff6(x, y)
    assert dp < 1e-6 and dr < 1e-6, (dp, dr)
    st = s.cholesky_stats()
    assert st["factorizations"] == r.iterations and st["failed_factorizations"] == 0 and st["factor_ms"] > 0
    s.close()
    h = pgo.pose_graph_to_4d(small_graph(seed=22, n=60, loops=150), seed=22)
    s = device(h, 4)
    s.solve()
    x4 = s.get_poses_4d(h["ids"])
    y4, _ = p4.solve_4d(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"], iters=60, ftol=1e-15)
    assert np.abs(x4[:, :3] - y4[:, :3]).max() < 1e-6 and np.abs(pgo.normalize_angle(x4[:, 3] - y4[:, 3])).max() < 1e-6
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
@pytest.mark.parametrize("params", list(tpa.SHIPPED))
def test_arock_with_cholesky_local_solves_matches_the_oracle(dof, params):
    gg = tpa.graph(dof)
    cfg = tpa.SHIPPED[params]
    # local solves to convergence: no function-tolerance stop, LM runs until no step lowers the cost.  Agents 1 and 2 hold
    # their gauge through the proximal terms alone; along that flat direction a step of ~1e-6 m changes the cost by less than
    # 1e-15 relative, so a 1e-15 function tolerance can stop that far from the optimum, wherever the step sequence ends
    kw = dict(linear_solver="sparse_cholesky", max_iterations=200, lambda0=1e-8, function_tolerance=0.0)
    dev = tpa.device_agents(gg, cfg, solver_kw=kw)
    orc = tpa.oracle_agents(gg, cfg)
    for r in range(10):
        pgo.arock_run(dev, 1); ao.arock_run(orc, 1)
        for d, o in zip(dev, orc):
            dp, dr = tpa.pose_diff(dof, d.poses(), o.x)
            assert dp < 1e-6 and dr < 1e-6, (r, d.self_id, dp, dr)
            assert d.s.cholesky_stats()["factorizations"] > 0
    for a in dev:
        a.close()


@pytest.mark.gpu
def test_solves_are_bitwise_reproducible_and_switching_back_is_pcg():
    g = with_extras(small_graph(seed=31), repeat=5, selfs=3)
    runs = []
    for _ in range(2):
        s = device(g, 6)
        r = s.solve(); runs.append((r.final_cost, s.get_poses(g["ids"]))); s.close()
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1])
    a = device(g, 6, max_iterations=5)
    a.solve()
    a.set_linear_solver("pcg")
    a.set_poses(g["ids"], g["init"], g["fixed"]); a.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    ra = a.solve(); xa = a.get_poses(g["ids"])
    b = device(g, 6, linear_solver="pcg", max_iterations=5)
    rb = b.solve(); xb = b.get_poses(g["ids"])
    assert ra.pcg_iterations == rb.pcg_iterations and ra.final_cost == rb.final_cost and np.array_equal(xa, xb)
    a.close(); b.close()


@pytest.mark.gpu
def test_refusals():
    from d2slam_b200 import solver
    L = pgo._lib()
    g = small_graph(seed=41, n=20, loops=30)
    s = device(g, 6, linear_solver="pcg")
    assert L.d2pgo_set_linear_solver(s.h, 7) == 2 and "unknown kind" in L.d2pgo_last_error(s.h).decode()
    s.set_linear_solver("sparse_cholesky")
    assert L.d2pgo_comm_init(s.h, (C.c_uint8 * 128)(*solver.comm_unique_id()), 0, 1) == 5   # Cholesky first, then a communicator
    s.close()
    s = device(g, 6, linear_solver="pcg")
    s.comm_init(solver.comm_unique_id(), 0, 1)
    assert L.d2pgo_set_linear_solver(s.h, 1) == 5                                          # a communicator first
    r = s.solve()                                                                          # still the PCG path
    assert r.pcg_iterations > 0
    s.close()


@pytest.mark.gpu
def test_an_oversized_front_is_refused_before_any_device_work():
    n = 400                                              # every pair joined: one front of 399 x 6 rows
    rng = np.random.default_rng(0)
    x = np.zeros((n, 7)); x[:, :3] = rng.normal(size=(n, 3)); x[:, 6] = 1.0
    a, b = np.triu_indices(n, 1)
    rel = pgo.relative_pose(x[a], x[b]); si = np.tile(np.eye(6).ravel(), (len(a), 1))
    fixed = np.zeros(n, np.uint8); fixed[0] = 1
    s = pgo.PgoSolver(linear_solver="sparse_cholesky")
    s.set_poses(np.arange(n), x, fixed); s.add_edges(a, b, rel, si)
    with pytest.raises(RuntimeError, match="front of"):
        s.solve()
    assert s.cholesky_stats()["max_front_rows"] > 1024 and s.cholesky_stats()["factorizations"] == 0
    assert np.array_equal(s.get_poses(np.arange(n)), x)
    s.close()


@pytest.mark.gpu
def test_a_free_component_without_a_fixed_pose_at_zero_damping():
    g = small_graph(seed=51, n=25, loops=40)
    h = small_graph(seed=52, n_agents=1, n=20, loops=10)   # a second component, nothing fixed in it
    ids = np.r_[g["ids"], h["ids"] + 10_000_000]
    m = dict(ids=ids, init=np.r_[g["init"], h["init"]], fixed=np.r_[g["fixed"], np.zeros(len(h["ids"]), np.uint8)],
             id_a=np.r_[g["id_a"], h["id_a"] + 10_000_000], id_b=np.r_[g["id_b"], h["id_b"] + 10_000_000],
             rel=np.r_[g["rel"], h["rel"]], sqrt_info=np.r_[g["sqrt_info"], h["sqrt_info"]])
    s = device(m, 6, lambda0=0.0)
    r = s.solve()
    x = s.get_poses(ids)
    assert np.all(np.isfinite(x)) and r.final_cost <= r.initial_cost
    s.close()
