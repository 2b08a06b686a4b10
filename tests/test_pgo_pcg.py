"""The pose graph's block-Jacobi PCG (the default linear solver of d2pgo_solve, of ARock's local solves and of d2pgo_rot_init's
row systems) as a linear solver, iterate by iterate, against a long-double restatement with the device's conventions, applied
record by record to the handle's own edge, gravity-prior and proximal-term records (include/d2pgo.h d2pgo_debug_pcg_step).

The restatement: dx = 0, r = -g, p = 0 over the free poses; M_i = (D_i + diag(lambda diag D_i + 1e-12))^-1 with D_i the sum of
J^T J over pose i's incidence entries (a self loop adds J0^T J0 + J1^T J1, not its true diagonal block); beta = rz / rz_prev
(0 first), alpha = rz / pAp (0 when pAp <= 0); stop before an iteration when rr <= tol^2 bb, rz <= 0 or rz is not finite, and
never run more than max_it iterations.  The device's iterates differ from it by the rounding of float64 sums, which CG
amplifies; how much is measured per case by e64, the largest distance of float64 restatements in different summation orders
from the long-double one, and the device must stay within max(10 e64, 64 eps |dx|).  CPU tests show that the restatement
solves small systems and that each of a set of plausible slips in a float64 copy of it breaks that check."""
import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pgo_arock_oracle as ao
from oracle import pgo_gravity_oracle as go
from oracle import pgo_lsq
from oracle import pgo_oracle as po
from oracle import pgo_rotinit_oracle as ro

import test_pgo_arock as tpa
import test_pgo_cholesky as tpc
import test_pgo_rotinit as tpr

LD = np.longdouble
EPS = np.finfo(float).eps
LAMBDAS = (0.0, 1e-4, 1.0, 1e4)
ITERATES = (1, 2, 3, 8, 16, 17, 33)        # around the 16-iteration chunks the device launches CG in
CAPS = (0, 1, 15, 16, 17, 31, 32, 33, 200)
SLIPS = ("no_damping_in_Ap", "lambda_times_one", "stale_beta", "extra_terms_only_in_D", "drop_last_edge", "extra_iteration")


# ------------------------------------------------------------------------------------------------ the restatement
def _inv(M):
    """inverses of SPD blocks [n, D, D] in M's dtype by Gauss-Jordan (numpy's linalg has no long double)"""
    D = M.shape[1]
    A = np.concatenate([M, np.broadcast_to(np.eye(D, dtype=M.dtype), M.shape)], axis=2)
    for j in range(D):
        A[:, j] /= A[:, j, j][:, None]
        for i in range(D):
            if i != j:
                A[:, i] -= A[:, i, j][:, None] * A[:, j]
    return A[:, :, D:]


class System:
    """(J^T J + diag(lam diag D + 1e-12)) dx = -g over the free poses, from factor records (test_pgo_cholesky.records'
    layout), every operation in dtype dt.  perm: a permutation of each group's records (another summation order); slips:
    deliberate departures from the device (SLIPS)."""

    def __init__(self, factors, fixed, D, lam, dt=LD, perm=None, slips=()):
        self.fixed = np.asarray(fixed) != 0; self.D = D; self.dt = dt; self.slips = set(slips)
        N = len(self.fixed)
        self.fac = []
        for k, (poses, r, Js) in enumerate(factors):
            o = np.arange(len(r)) if perm is None else perm(len(r))
            self.fac.append(([np.asarray(c)[o] for c in poses], np.asarray(r)[o].astype(dt), [np.asarray(J)[o].astype(dt) for J in Js]))
        self.g = np.zeros((N, D), dt); Db = np.zeros((N, D, D), dt)
        for poses, r, Js in self.fac:
            for c, J in zip(poses, Js):
                np.add.at(self.g, c, np.einsum("emd,em->ed", J, r))
                np.add.at(Db, c, np.einsum("emd,emf->edf", J, J))
        self.g[self.fixed] = 0; Db[self.fixed] = 0
        dg = np.einsum("ndd->nd", Db)
        self.damp = (dt(lam) * (np.ones_like(dg) if "lambda_times_one" in self.slips else dg) + dt(1e-12)) * ~self.fixed[:, None]
        self.Minv = np.zeros_like(Db)
        free = ~self.fixed
        self.Minv[free] = _inv(Db[free] + np.einsum("nd,de->nde", self.damp[free], np.eye(D, dtype=dt)))
        self.drop = None
        if "drop_last_edge" in self.slips:   # one free pose with two or more edges misses the last one in its product sum
            ea, eb = self.fac[0][0]
            inc = lambda i: (ea == i) ^ (eb == i)   # a self loop near the identity has J0 = -J1 and no product to miss
            i = next(i for i in np.nonzero(free)[0] if inc(i).sum() >= 2)
            self.drop = (i, np.nonzero(inc(i))[0].max())

    def Ap(self, p):
        y = np.zeros_like(p)
        for k, (poses, _, Js) in enumerate(self.fac):
            if k > 0 and "extra_terms_only_in_D" in self.slips:
                continue
            t = sum(np.einsum("emd,ed->em", J, p[c]) for c, J in zip(poses, Js))
            for c, J in zip(poses, Js):
                yc = np.einsum("emd,em->ed", J, t)
                if k == 0 and self.drop is not None:
                    yc[(c == self.drop[0]) & (np.arange(len(c)) == self.drop[1])] = 0
                np.add.at(y, c, yc)
        y[self.fixed] = 0
        return y if "no_damping_in_Ap" in self.slips else y + self.damp * p

    def M(self, r):
        return np.einsum("nde,ne->nd", self.Minv, r)


def pcg(S, tol, max_it, keep=()):
    """the device's PCG on system S: (dx, iterations, sqrt(rr / bb) of the last update, rr / bb after each iteration (index 0:
    the start), {k: dx after k iterations for k in keep})"""
    dt = S.dt
    dx = np.zeros_like(S.g); r = -S.g; z = S.M(r); p = np.zeros_like(S.g)
    rz = np.sum(r * z); rr = np.sum(r * r); bb = rr
    rzs = [rz]; ratios = [rr / bb if bb > 0 else dt(0)]; snaps = {}
    it = 0
    n = max_it + ("extra_iteration" in S.slips)
    while it < n:
        if not (rr > dt(tol) * dt(tol) * bb) or not (rz > 0) or not np.isfinite(rz):
            break
        if it == 0:
            beta = dt(0)
        elif "stale_beta" in S.slips:
            beta = rzs[it - 1] / rzs[max(it - 2, 0)]
        else:
            beta = rzs[it] / rzs[it - 1]
        p = z + beta * p
        q = S.Ap(p)
        pAp = np.sum(p * q)
        alpha = rz / pAp if pAp > 0 else dt(0)
        dx = dx + alpha * p; r = r - alpha * q; z = S.M(r)
        rz = np.sum(r * z); rr = np.sum(r * r); rzs.append(rz); ratios.append(rr / bb)
        it += 1
        if it in keep:
            snaps[it] = dx.copy()
    for k in keep:                                       # stopped early: later counts keep the last iterate
        snaps.setdefault(k, dx.copy())
    return dx, it, float(np.sqrt(rr / bb)) if bb > 0 else 0.0, np.array(ratios, dtype=float), snaps


ORDERS = {"natural": None, "reversed": lambda n: np.arange(n)[::-1], "shuffled": lambda n: np.random.default_rng(n).permutation(n)}


def reference_iterates(factors, fixed, D, lam, counts):
    """{k: dx_LD after k iterations} and {k: e64}, tol = 0"""
    ld = pcg(System(factors, fixed, D, lam), 0.0, max(counts), counts)[4]
    e64 = {k: 0.0 for k in counts}
    for perm in ORDERS.values():
        s64 = pcg(System(factors, fixed, D, lam, np.float64, perm), 0.0, max(counts), counts)[4]
        for k in counts:
            e64[k] = max(e64[k], float(np.abs(s64[k] - ld[k]).max(initial=0.0)))
    return ld, e64


def iterate_ratio(dx, ld, e64):
    """|dx - dx_LD|_inf over the check-1 bound max(10 e64, 64 eps |dx_LD|_inf); 0 when both sides are 0"""
    err = float(np.abs(np.asarray(dx, float) - np.asarray(ld, float)).max(initial=0.0))
    bound = max(10 * e64, 64 * EPS * float(np.abs(ld).max(initial=0.0)))
    return err / bound if bound > 0 else (0.0 if err == 0 else np.inf)


# ------------------------------------------------------------------------------------------------ CPU
def oracle_factors(dof=6, priors=False, prox=False, seed=3, n=12, loops=30):
    """oracle records (pgo_oracle.edges_eval, pgo4d_oracle, gravity and proximal terms) of a small graph with duplicate edges,
    self loops and a second fixed pose: (factors, fixed)"""
    g = tpc.with_extras(tpc.small_graph(seed=seed, n=n, loops=loops), repeat=4, selfs=3)
    if dof == 4:
        g = tpc.with_extras(pgo.pose_graph_to_4d(tpc.small_graph(seed=seed, n=n, loops=loops), seed=seed), repeat=4, selfs=3)
    fixed = np.array(g["fixed"]); fixed[n + 1] = 1
    x = np.asarray(g["init"]); ea, eb = np.asarray(g["ea"]), np.asarray(g["eb"])
    if dof == 4:
        from oracle import pgo4d_oracle as p4
        r, J0, J1 = p4.edges_eval_4d(x, ea, eb, np.asarray(g["rel"]), np.asarray(g["sqrt_info"]).reshape(-1, 4, 4))
    else:
        r, J0, J1 = po.edges_eval(x, ea, eb, np.asarray(g["rel"]), np.asarray(g["sqrt_info"]).reshape(-1, 6, 6))
    factors = [((ea, eb), r, (J0, J1))]
    N = len(x)
    if priors:
        idx = np.arange(0, N, 2)
        ego = pgo.make_gravity_case(g, seed=seed)["ego"][idx]
        rg, Jg = go.priors_eval(x, idx, go.ego_gravity(ego), np.tile(pgo.GRAVITY_SQRT_INFO * np.eye(3), (len(idx), 1, 1)))
        factors.append(((idx,), rg, (Jg,)))
    if prox:
        idx = np.arange(1, N, 3)
        rng = np.random.default_rng(seed)
        y = ao.coords(x[idx], x[idx, 3:7] if dof == 6 else None) + rng.normal(0, 0.05, (len(idx), dof))
        rp, Jp = ao.prox_eval(x[idx], x[idx, 3:7] if dof == 6 else None, y, 0.7, 0.625)
        factors.append(((idx,), rp, (Jp,)))
    return factors, fixed


def test_restatement_reaches_the_dense_solve():
    for dof, priors, prox in ((6, True, True), (4, False, True), (6, False, False)):
        factors, fixed = oracle_factors(dof, priors, prox)
        for lam in LAMBDAS:
            A, b, _ = tpc.assemble(None, dict(fixed=fixed), dof, lam, factors=factors)
            ref = np.linalg.solve(A.toarray(), b)
            dx, it, res, _, _ = pcg(System(factors, fixed, dof, lam), 1e-15, 5000)
            x = np.asarray(dx, float)[fixed == 0].ravel()
            assert res <= 1e-15 and it < 5000
            assert np.abs(x - ref).max() <= 1e-9 * np.abs(ref).max(), (dof, lam, np.abs(x - ref).max())
            assert np.all(dx[fixed != 0] == 0)


@pytest.mark.parametrize("slip", SLIPS)
def test_each_slip_breaks_the_iterate_check(slip):
    """a float64 copy of the restatement with one slip, standing in for the device, fails check 1 somewhere; without it,
    every float64 order passes (it is one of the orders e64 is taken over)"""
    worst = 0.0
    for dof in (6, 4):
        factors, fixed = oracle_factors(dof, priors=dof == 6, prox=True)
        for lam in LAMBDAS:
            ld, e64 = reference_iterates(factors, fixed, dof, lam, ITERATES)
            bad = pcg(System(factors, fixed, dof, lam, np.float64, slips=(slip,)), 0.0, max(ITERATES), ITERATES)[4]
            for k in ITERATES:
                if slip == "extra_iteration":   # the cap defect: every count runs one iteration more
                    bad[k] = pcg(System(factors, fixed, dof, lam, np.float64, slips=(slip,)), 0.0, k)[0]
                worst = max(worst, iterate_ratio(bad[k], ld[k], e64[k]))
    print(f"{slip}: largest |dx - dx_LD| / bound {worst:.3g}")
    assert worst > 1.0, slip


def test_all_fixed_and_zero_gradient_give_no_iterations():
    factors, fixed = oracle_factors(6)
    dx, it, res, _, _ = pcg(System(factors, np.ones_like(fixed), 6, 1.0), 0.0, 33)
    assert it == 0 and res == 0.0 and np.all(dx == 0)


# ------------------------------------------------------------------------------------------------ GPU cases
def _full_sqrt_info(g, seed):
    """random upper-triangular-plus-noise 6x6 square roots of information (every entry non-zero)"""
    rng = np.random.default_rng(seed)
    E = len(g["ea"])
    S = rng.normal(0, 2.0, (E, 6, 6)) + np.diag([20.0, 20.0, 20.0, 57.0, 57.0, 57.0])[None]
    return dict(g, sqrt_info=S.reshape(E, 36))


def _with_lonely_pose(g):
    """one more free pose that no edge names"""
    p = np.asarray(g["init"])[-1:].copy(); p[0, 0] += 1.0
    return dict(g, ids=np.r_[g["ids"], 77_000_000], init=np.r_[g["init"], p], fixed=np.r_[g["fixed"], 0].astype(np.uint8))


def _sized(n_free, n_edges, seed):
    """one agent, pose 0 fixed and n_free free, the first n_edges edges (odometry first)"""
    g = pgo.make_pose_graph(seed=seed, n_agents=1, poses_per_agent=n_free + 1, loops=2 * n_edges)
    E = min(n_edges, len(g["ea"]))
    return dict(g, ea=g["ea"][:E], eb=g["eb"][:E], id_a=g["id_a"][:E], id_b=g["id_b"][:E], rel=g["rel"][:E], sqrt_info=g["sqrt_info"][:E])


def case(name):
    """dict(s = a PCG handle, dof, fixed, factors = its records, closers)"""
    ego, dof, prior_idx = None, 6, None
    if name == "6dof_full_sqrt_info":
        g = tpc.with_extras(_full_sqrt_info(tpc.small_graph(seed=61, n=30, loops=80), 61), repeat=8, selfs=4)
        g = _with_lonely_pose(g)
        g["fixed"] = g["fixed"].copy(); g["fixed"][[0, 45]] = 1      # edges with a fixed pose at either end
    elif name == "4dof_yaw_wrap":
        h = tpa.rotate4(pgo.pose_graph_to_4d(tpc.small_graph(seed=62, n=30, loops=80), seed=62), np.pi - 0.05)
        g = tpc.with_extras(h, repeat=8, selfs=4)
        g["fixed"] = g["fixed"].copy(); g["fixed"][[0, 45]] = 1
        dof = 4
    elif name in ("6dof_gravity_all", "6dof_gravity_subset"):
        g = tpc.with_extras(tpc.small_graph(seed=63, n=30, loops=80), repeat=4, selfs=2)
        ego = pgo.make_gravity_case(g, seed=63)["ego"]
        prior_idx = np.arange(len(g["ids"])) if name.endswith("all") else np.arange(0, len(g["ids"]), 3)
    elif name.startswith("free_"):
        n, e = {"free_1": (1, 1), "free_127": (127, 255), "free_128": (128, 256), "free_129": (129, 257), "free_1000": (1000, 3841)}[name]
        g = _sized(n, e, seed=64 + n)
    elif name == "all_fixed":
        g = tpc.small_graph(seed=65, n=10, loops=20)
        g["fixed"] = np.ones(len(g["ids"]), np.uint8)
    elif name == "bench":
        g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
    elif name.startswith("arock"):
        dof = int(name[-1])
        agents = tpa.device_agents(tpa.graph(dof), tpa.SHIPPED["default"])
        pgo.arock_run(agents, 1)
        a = agents[0]; sp_ = a.split
        pos = {int(i): k for k, i in enumerate(sp_["ids"])}
        gg = dict(ids=sp_["ids"], fixed=sp_["fixed"], ea=np.array([pos[int(i)] for i in sp_["id_a"]]), eb=np.array([pos[int(i)] for i in sp_["id_b"]]))
        arock_poses = [pos[f] for _, f in sorted(a.duals())]
        assert arock_poses
        return dict(s=a.s, dof=dof, fixed=np.asarray(gg["fixed"]), factors=tpc.records(a.s, gg, dof, arock_poses=arock_poses), closers=agents)
    else:
        raise KeyError(name)
    s = pgo.PgoSolver(pose_dof=dof)
    if dof == 4:
        s.set_poses_4d(g["ids"], g["init"], g["fixed"]); s.add_edges_4d(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    else:
        s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    factors = tpc.records(s, g, dof)
    if ego is not None:
        s.add_gravity_priors(g["ids"][prior_idx], ego[prior_idx])
        pr = s.debug_gravity_priors()
        factors.append(((prior_idx,), pr[:, :3], (pr[:, 3:].reshape(-1, 3, 6),)))
    return dict(s=s, dof=dof, fixed=np.asarray(g["fixed"]), factors=factors, closers=[s], g=g)


def close(c):
    for x in c["closers"]:
        x.close()


CASES = ["6dof_full_sqrt_info", "4dof_yaw_wrap", "6dof_gravity_all", "6dof_gravity_subset", "arock4", "arock6",
         "free_1", "free_127", "free_128", "free_129", "free_1000"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES + ["bench"])
def test_iterates_match_the_long_double_restatement(name):
    c = case(name)
    counts = (16, 17) if name == "bench" else ITERATES
    lams = (1e-4,) if name == "bench" else LAMBDAS
    worst = 0.0
    for lam in lams:
        ld, e64 = reference_iterates(c["factors"], c["fixed"], c["dof"], lam, counts)
        ratios = pcg(System(c["factors"], c["fixed"], c["dof"], lam), 0.0, max(counts))[3]
        for k in counts:
            dx, it, _ = c["s"].debug_pcg_step(lam, k, 0.0)
            # an earlier stop (rz <= 0 or rr = 0 in float64) only once the system is solved to rounding
            assert it == k or (it < k and ratios[it] < (64 * EPS) ** 2), (name, lam, k, it)
            assert np.all(dx[c["fixed"] != 0] == 0)
            q = iterate_ratio(dx, ld[k], e64[k])
            worst = max(worst, q)
            assert q <= 1.0, (name, lam, k, q, e64[k])
    print(f"{name}: largest |dx_dev - dx_LD| / bound {worst:.3g}")
    close(c)


@pytest.mark.gpu
def test_all_fixed_poses_give_zero_iterations_and_zero_step():
    c = case("all_fixed")
    for lam in LAMBDAS:
        dx, it, res = c["s"].debug_pcg_step(lam, 33, 0.0)
        assert it == 0 and res == 0.0 and np.all(dx == 0), (lam, it, res)
    close(c)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof_gravity_subset", "arock4"])
def test_the_iteration_cap_is_exact(name):
    """iterations = the cap, and the residual of the last update the restatement's to 1e-6 or to 10 times the spread of the
    float64 orders' (long runs amplify rounding)"""
    c = case(name)
    lam = 1e-4
    ref = pcg(System(c["factors"], c["fixed"], c["dof"], lam), 0.0, max(CAPS))[3]
    r64 = [pcg(System(c["factors"], c["fixed"], c["dof"], lam, np.float64, p), 0.0, max(CAPS))[3] for p in ORDERS.values()]
    for k in CAPS:
        dx, it, res = c["s"].debug_pcg_step(lam, k, 0.0)
        assert it == k or (it < k and ref[it] < (64 * EPS) ** 2), (name, k, it)
        want = float(np.sqrt(ref[k]))
        spread = max(abs(np.sqrt(r[min(k, len(r) - 1)]) - want) for r in r64)
        assert abs(res - want) <= max(1e-6 * want, 10 * spread), (name, k, res, want, spread)
    close(c)


@pytest.mark.gpu
def test_an_lm_iteration_stops_at_pcg_max_iterations():
    g = tpc.small_graph(seed=66, n=30, loops=80)
    s = pgo.PgoSolver(max_iterations=1, pcg_max_iterations=20, pcg_tolerance=0.0, lambda0=1e-4)
    s.set_poses(g["ids"], g["init"], g["fixed"]); s.add_edges(g["id_a"], g["id_b"], g["rel"], g["sqrt_info"])
    factors = tpc.records(s, g, 6)
    r = s.solve()
    assert (r.iterations, r.pcg_iterations) == (1, 20), (r.iterations, r.pcg_iterations)
    dx = np.asarray(pcg(System(factors, g["fixed"], 6, 1e-4), 0.0, 20)[0], float)
    free = np.nonzero(g["fixed"] == 0)[0]
    assert r.accepted == 1
    want = pgo_lsq.retract(np.asarray(g["init"]), free, dx[free].ravel())
    dp, dr = tpc.pose_diff6(s.get_poses(g["ids"]), want)
    assert dp < 1e-9 and dr < 1e-9, (dp, dr)
    s.close()


def rot_row_factors(sys_, k):
    """row system k of the chordal relaxation (oracle build_system) as factor records over the free frames: each 3-row block
    of A's rows in the columns of R_f's row k, with r = -b so that sum J^T r = -A_k^T b_k"""
    A, b = sys_["A"].tocsr(), sys_["b"]
    F = len(sys_["frames"])
    cols = (9 * np.arange(F)[:, None] + 3 * k + np.arange(3)).ravel()
    Ak = A[:, cols].tocsr()
    rows = np.nonzero(np.diff(Ak.indptr) > 0)[0].reshape(-1, 3)
    assert np.all(rows == rows[:, :1] + np.arange(3))
    dense = Ak[rows.ravel()].toarray().reshape(len(rows), 3, F, 3)
    touched = [np.nonzero(np.abs(dense[t]).sum(axis=(0, 2)) > 0)[0] for t in range(len(rows))]
    r = -b[rows]
    out = []
    for m in (2, 1):
        sel = np.array([t for t in range(len(rows)) if len(touched[t]) == m], int)
        if len(sel):
            poses = tuple(np.array([touched[t][j] for t in sel]) for j in range(m))
            out.append((poses, r[sel], tuple(dense[sel, :, poses[j], :] for j in range(m))))
    assert sum(len(f[1]) for f in out) == len(rows)
    return out, F


@pytest.mark.gpu
@pytest.mark.parametrize("gravity", [False, True])
def test_rot_init_rows_stop_at_the_cap(gravity):
    c = tpr.graph_case(67, n_agents=3, n=40, loops=100, tilt=0.4, gravity=gravity, quirk=True, self_loop=True)
    s = tpr._solver(c)
    rep = tpr._rot_init(s, c, pcg_max_iterations=20, pcg_tolerance=0.0)
    sys_ = ro.build_system(c["ids"], c["poses"], c["fixed"], c["id_a"], c["id_b"], c["rel"], c["sqrt_info"], gravity,
                           pgo.GRAVITY_SQRT_INFO, c["ego_ids"], c["ego"])
    for k in range(3):
        factors, F = rot_row_factors(sys_, k)
        _, it, res, _, _ = pcg(System(factors, np.zeros(F, np.uint8), 3, 0.0), 0.0, 20)
        assert it == 20 and rep["pcg_iterations"][k] == 20, (k, rep["pcg_iterations"])
        assert abs(rep["residual"][k] - res) <= 1e-6 * res, (k, rep["residual"][k], res)
    s.close()


def kappa(A):
    w = np.linalg.eigvalsh(A.toarray())
    return float(w[-1] / w[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof_full_sqrt_info", "4dof_yaw_wrap", "6dof_gravity_all", "arock6", "free_129"])
def test_convergence_to_the_tolerance(name):
    """the stop count is the restatement's (one off only where the float64 orders disagree about which side of tol^2 the
    recurrence is), the returned residual is below tol, the true residual |A dx + g| below 2 tol |g| plus what float64 cannot
    resolve: the device's own g and A differ from the records' exact sums by eps times the sums of magnitudes (at a converged
    ARock agent g cancels to ~1e-8 of its terms), and the CG recurrence drifts from the true residual by about eps times that
    per iteration; at 1e-10, dx is the exact step's to kappa times the residual reached"""
    c = case(name)
    D = c["dof"]
    free = c["fixed"] == 0
    for lam in LAMBDAS:
        S = System(c["factors"], c["fixed"], D, lam)
        A, b, k_terms = tpc.assemble(None, dict(fixed=c["fixed"]), D, lam, factors=c["factors"])
        Am, bm, _ = tpc.assemble(None, dict(fixed=c["fixed"]), D, lam, factors=c["factors"], magnitude=True)
        b = -np.asarray(S.g, float)[free].ravel()
        for tol in (1e-2, 1e-6, 1e-10):
            dx, it, res = c["s"].debug_pcg_step(lam, 5000, tol)
            _, it_ld, _, ratios, _ = pcg(S, tol, 5000)
            if it != it_ld:
                # one off where the recurrence ends within 1e-6 of tol^2; else within one of the float64 orders' own counts,
                # which spread where the residual reaches its rounding floor (tol 1e-10 at lambda 0)
                its = [it_ld] + [pcg(System(c["factors"], c["fixed"], D, lam, np.float64, p), tol, 5000)[1] for p in ORDERS.values()]
                j = min(it, it_ld)
                near = abs(it - it_ld) == 1 and abs(ratios[j] - tol * tol) <= 1e-6 * tol * tol
                assert near or min(its) - 1 <= it <= max(its) + 1, (name, lam, tol, it, its)
            assert res <= tol, (name, lam, tol, res)
            true = _residual(A, dx[free].ravel(), b)
            unc = (k_terms * D + 2) * EPS * ((it + 1) * np.linalg.norm(Am @ np.abs(dx[free].ravel())) + np.linalg.norm(bm))
            assert true <= 2 * tol * np.linalg.norm(b) + unc, (name, lam, tol, true / np.linalg.norm(b), unc / np.linalg.norm(b))
            if tol == 1e-10:
                ex = c["s"].debug_exact_step(lam)[free].ravel()
                k = kappa(A)
                err = np.linalg.norm(dx[free].ravel() - ex) / np.linalg.norm(ex)
                rel = true / np.linalg.norm(b)
                print(f"{name} lambda {lam:g}: {it} iterations, true residual {rel:.2e}, kappa {k:.2e}, |dx - dx_exact| / |dx_exact| {err:.2e}")
                assert err <= k * max(2 * tol, rel), (name, lam, err, k)
    close(c)


def _residual(A, x, b):
    """|A x - b|_2 with the products and sums in long double (b = -g)"""
    A = A.tocsr()
    prod = A.data.astype(LD) * x.astype(LD)[A.indices]
    Ax = np.zeros(A.shape[0], LD)
    nz = np.diff(A.indptr) > 0
    Ax[nz] = np.add.reduceat(prod, A.indptr[:-1][nz])
    return float(np.sqrt(np.sum((Ax - b.astype(LD)) ** 2)))


@pytest.mark.gpu
def test_bench_settings_stop_where_the_restatement_stops():
    c = case("bench")
    lam = 1e-4
    dx, it, res = c["s"].debug_pcg_step(lam, 200, 1e-1)
    _, it_ld, res_ld, ratios, _ = pcg(System(c["factors"], c["fixed"], 6, lam), 1e-1, 200)
    print(f"bench: {it} iterations (restatement {it_ld}), residual {res:.4g} ({res_ld:.4g})")
    assert it == it_ld and res <= 1e-1 and abs(res - res_ld) <= 1e-6 * res_ld
    close(c)


@pytest.mark.gpu
def test_captured_graphs_are_reused_only_for_the_same_chunk():
    """one handle called with 17, 33, 17 iterations and then another tolerance gives bitwise what fresh handles give"""
    calls = [(1e-4, 17, 0.0), (1e-4, 33, 0.0), (1e-4, 17, 0.0), (1e-4, 33, 1e-3), (1.0, 17, 0.0)]
    c = case("6dof_gravity_subset")
    one = [c["s"].debug_pcg_step(*a) for a in calls]
    close(c)
    for a, (dx, it, res) in zip(calls, one):
        f = case("6dof_gravity_subset")
        dx2, it2, res2 = f["s"].debug_pcg_step(*a)
        close(f)
        assert it == it2 and res == res2 and np.array_equal(dx, dx2), a


@pytest.mark.gpu
def test_refusals():
    import ctypes as C
    from d2slam_b200 import solver
    L = pgo._lib()
    c = case("free_1")
    s = c["s"]
    out = np.zeros((2, 6)); it = C.c_int32(); res = C.c_double()

    def call(lam=0.0, k=4, tol=0.0, buf=out, n=None, itp=True):
        return L.d2pgo_debug_pcg_step(s.h, C.c_double(lam), C.c_int32(k), C.c_double(tol), pgo._p(buf), C.c_int64(buf.size if n is None else n),
                                      C.byref(it) if itp else None, C.byref(res))
    assert call() == 0
    assert call(itp=False) == 1
    assert L.d2pgo_debug_pcg_step(s.h, C.c_double(0.0), C.c_int32(4), C.c_double(0.0), None, C.c_int64(12), C.byref(it), C.byref(res)) == 1
    assert call(n=11) == 2 and "too small" in L.d2pgo_last_error(s.h).decode()
    for bad in (dict(lam=-1.0), dict(lam=float("nan")), dict(lam=float("inf")), dict(tol=-1e-3), dict(tol=float("nan")), dict(k=-1)):
        assert call(**bad) == 2, bad
    s.comm_init(solver.comm_unique_id(), 0, 1)
    assert call() == 5
    close(c)
