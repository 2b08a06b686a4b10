"""CPU oracle of the pose graph's ceres minimiser (TEST INFRASTRUCTURE: imported by tests/ and tools/ only).

Restates d2pgo_set_minimizer(h, D2PGO_MINIMIZER_CERES_LM, cfg) (include/d2pgo.h): ceres 2.1's TrustRegionMinimizer with
LevenbergMarquardtStrategy, the linear solve replaced by scipy's sparse direct solver (what the sparse Cholesky computes):
  start     r, J, d at x0 (pgo_lm_oracle.Problem.system: d = the diagonal of the per-pose block diagonal); Jacobi scale
            s = 1 / (1 + sqrt(d)) once (1 without jacobi_scaling); gradient test max |x - x [+] (-g)| <= gradient_tolerance
            over the free poses' ambient components
  iteration stop when the count of accepted and rejected steps reaches max_num_iterations; solve
            (J^T J + diag(mu)) dx = -g, mu = clamp(s^2 d, min_lm_diagonal, max_lm_diagonal) / (radius s^2)
  model     m = -(r.(J dx) + |J dx|^2 / 2); invalid when m <= 0 or anything is non-finite (rejected; FAILURE after more than
            max_num_consecutive_invalid_steps in a row)
  tests     parameter |dx| <= ptol (|x| + ptol), then function |C - C+| <= ftol C (both return x), then accept on
            rho = (C - C+) / m > min_relative_decrease: radius = min(radius / max(1/3, 1 - (2 rho - 1)^3), max radius),
            decrease factor 2, relinearise, gradient test; else radius /= decrease factor, decrease factor *= 2, stop when
            radius < min_trust_region_radius
The time budget (max_solver_time_in_seconds) is the device's clock and is not restated here.  The points marked ASSUMED in
include/d2pgo.h are defined by this file; the device matches it."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import pgo_lsq

DEFAULTS = dict(max_num_iterations=50, max_num_consecutive_invalid_steps=5, jacobi_scaling=1, max_solver_time_in_seconds=0.0,
                initial_trust_region_radius=1e4, max_trust_region_radius=1e16, min_trust_region_radius=1e-32,
                min_relative_decrease=1e-3, min_lm_diagonal=1e-6, max_lm_diagonal=1e32, function_tolerance=1e-6,
                gradient_tolerance=1e-10, parameter_tolerance=1e-8)
ACCEPTED, REJECTED, INVALID, CONVERGED = 0, 1, 2, 3                 # step kinds (D2PGO_STEP_*)
CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2                      # termination types (D2PGO_TERMINATION_*)
GRADIENT, PARAMETER, FUNCTION, MIN_RADIUS, MAX_ITERATIONS, TIME, INVALID_STEPS = 1, 2, 3, 4, 5, 6, 7   # D2PGO_STOP_*


class BlocksProblem:
    """A pose graph given as pgo_lsq residual blocks: x0 [N, 4 or 7], fixed flags, blocks_at(x) -> [(r, [(idx, J), ...])].
    The same interface as pgo_lm_oracle.Problem (system, cost, retract, free)."""

    def __init__(self, x0, fixed, blocks_at):
        self.x0 = np.array(x0, np.float64)
        self.D = 4 if self.x0.shape[1] == 4 else 6
        self.fixed = np.asarray(fixed) != 0
        self.blocks_at = blocks_at
        self.free, self.col = pgo_lsq.free_columns(self.fixed, self.D)

    def system(self, x):
        return pgo_lsq.assemble(self.blocks_at(x), self.col, len(self.free), self.D, diag=True)

    def cost(self, x):
        r = self.system(x)[0]
        return 0.5 * float(r @ r)

    def retract(self, x, dx):
        return pgo_lsq.retract(x, self.free, dx)


class LmStrategy:
    """LevenbergMarquardtStrategy's radius and decrease factor."""

    def __init__(self, radius, max_radius):
        self.radius, self.max_radius, self.decrease_factor = float(radius), float(max_radius), 2.0

    def accepted(self, rho):
        t = 2.0 * rho - 1.0
        self.radius = min(self.radius / max(1.0 / 3.0, 1.0 - t * t * t), self.max_radius)
        self.decrease_factor = 2.0

    def rejected(self):
        self.radius = self.radius / self.decrease_factor
        self.decrease_factor = 2.0 * self.decrease_factor


def jacobi_scale(d, jacobi_scaling=1):
    return 1.0 / (1.0 + np.sqrt(d)) if jacobi_scaling else np.ones_like(d)


def damping(d, scale, radius, lo=1e-6, hi=1e32):
    s2 = scale * scale
    return np.clip(s2 * d, lo, hi) / (radius * s2)


def gradient_max_norm(prob, x, g):
    """max over the free poses' ambient components of |x - x [+] (-g)|"""
    if not len(prob.free):
        return 0.0
    return float(np.abs(x[prob.free] - prob.retract(x, -g)[prob.free]).max())


def ambient_norm(prob, x):
    return float(np.linalg.norm(x[prob.free]))


def lm_step(J, r, mu):
    """(J^T J + diag(mu)) dx = -J^T r by a sparse direct solve; non-finite entries mark a failed factorisation"""
    if not J.shape[1]:
        return np.zeros(0)
    H = (J.T @ J).tocsc() + sp.diags(mu, format="csc")
    return spla.spsolve(H, -(J.T @ r))


def model_cost_change(J, r, dx):
    f = J @ dx
    return -(float(r @ f) + 0.5 * float(f @ f))


def ceres_lm_solve(prob, **cfg):
    """The device's ceres minimiser.  Returns (x, trace, report): trace = list of dicts (cost, candidate_cost,
    model_cost_change, relative_decrease, step_norm, radius, decrease_factor, kind) per iteration, report = dict(type, reason,
    successful_steps, unsuccessful_steps, final_radius, initial_cost, final_cost, scale)."""
    c = dict(DEFAULTS)
    for k, v in cfg.items():
        if k not in c:
            raise KeyError(k)
        c[k] = v
    x = prob.x0.copy()
    r, J, d = prob.system(x)
    cost = 0.5 * float(r @ r); g = J.T @ r
    scale = jacobi_scale(d, c["jacobi_scaling"])
    lm = LmStrategy(c["initial_trust_region_radius"], c["max_trust_region_radius"])
    trace = []
    rep = dict(type=None, reason=None, successful_steps=0, unsuccessful_steps=0, initial_cost=cost, scale=scale)

    def record(cand, rho, m, step_norm, kind):
        trace.append(dict(cost=cost, candidate_cost=cand, model_cost_change=m, relative_decrease=rho, step_norm=step_norm,
                          radius=lm.radius, decrease_factor=lm.decrease_factor, kind=kind))
        rep["successful_steps" if kind == ACCEPTED else "unsuccessful_steps"] += 1

    def stop(t, why):
        rep["type"], rep["reason"] = t, why

    x_norm = ambient_norm(prob, x)
    if gradient_max_norm(prob, x, g) <= c["gradient_tolerance"]:
        stop(CONVERGENCE, GRADIENT)
    invalid_run = 0
    while rep["type"] is None:
        if len(trace) >= c["max_num_iterations"]:
            stop(NO_CONVERGENCE, MAX_ITERATIONS)
            break
        with np.errstate(all="ignore"):
            dx = lm_step(J, r, damping(d, scale, lm.radius, c["min_lm_diagonal"], c["max_lm_diagonal"]))
            m = model_cost_change(J, r, dx)
            step_norm = float(np.linalg.norm(dx))
        if not (np.all(np.isfinite(dx)) and np.isfinite(m) and m > 0.0 and np.isfinite(step_norm)):
            invalid_run += 1
            if invalid_run > c["max_num_consecutive_invalid_steps"]:
                record(np.nan, np.nan, m, step_norm, INVALID)
                stop(FAILURE, INVALID_STEPS)
            else:
                lm.rejected()
                record(np.nan, np.nan, m, step_norm, INVALID)
                if lm.radius < c["min_trust_region_radius"]:
                    stop(CONVERGENCE, MIN_RADIUS)
            continue
        invalid_run = 0
        if step_norm <= c["parameter_tolerance"] * (x_norm + c["parameter_tolerance"]):
            record(np.nan, np.nan, m, step_norm, CONVERGED)
            stop(CONVERGENCE, PARAMETER)
            break
        xc = prob.retract(x, dx)
        cc = prob.cost(xc)
        if not np.isfinite(cc):
            cc = np.finfo(np.float64).max
        dc = cost - cc
        rho = dc / m
        if abs(dc) <= c["function_tolerance"] * cost:
            record(cc, rho, m, step_norm, CONVERGED)
            stop(CONVERGENCE, FUNCTION)
            break
        if rho > c["min_relative_decrease"]:
            lm.accepted(rho)
            record(cc, rho, m, step_norm, ACCEPTED)
            x = xc
            r, J, d = prob.system(x)
            cost = 0.5 * float(r @ r); g = J.T @ r
            x_norm = ambient_norm(prob, x)
            if gradient_max_norm(prob, x, g) <= c["gradient_tolerance"]:
                stop(CONVERGENCE, GRADIENT)
        else:
            lm.rejected()
            record(cc, rho, m, step_norm, REJECTED)
            if lm.radius < c["min_trust_region_radius"]:
                stop(CONVERGENCE, MIN_RADIUS)
    rep["final_radius"] = lm.radius
    rep["final_cost"] = cost
    return x, trace, rep


def arock_local_solve(x, fixed, ea, eb, rel, S, dual_pose, q_init_d, yr, rho_T, rho_theta, priors=None, cfg=None):
    """pgo_arock_oracle.local_solve's problem (the agent's edges, gravity priors and proximal terms) minimised by
    ceres_lm_solve(**cfg) instead of Gauss-Newton to convergence.  Returns (poses, [initial cost, final cost])."""
    from oracle import pgo_arock_oracle as pa
    x = np.asarray(x, np.float64); D = 4 if x.shape[1] == 4 else 6
    ea = np.asarray(ea); eb = np.asarray(eb); rel = np.asarray(rel, np.float64)
    S = np.asarray(S, np.float64).reshape(-1, D, D); dual_pose = np.asarray(dual_pose, int)

    def blocks(x):
        r_e, J0, J1 = (pa.edges_eval_4d if D == 4 else pa.edges_eval)(x, ea, eb, rel, S)
        out = [(r_e, [(ea, J0), (eb, J1)])]
        if priors is not None and len(priors[0]):
            r_g, Jg = pa.priors_eval(x, priors[0], priors[1], priors[2])
            out.append((r_g, [(np.asarray(priors[0]), Jg)]))
        if len(dual_pose):
            r_k, J_k = pa.prox_eval(x[dual_pose], q_init_d, yr, rho_T, rho_theta)
            out.append((r_k, [(dual_pose, J_k)]))
        return out
    xs, _, rep = ceres_lm_solve(BlocksProblem(x, fixed, blocks), **(cfg or {}))
    return xs, [rep["initial_cost"], rep["final_cost"]]


def arock_agent(split, lm_cfg=None, **kw):
    """A pgo_arock_oracle.OracleAgent whose local solves run ceres_lm_solve(**lm_cfg) (d2pgo_arock_step on a handle with the
    ceres minimiser).  kw: OracleAgent's arguments."""
    from oracle import pgo_arock_oracle as pa

    class CeresLmAgent(pa.OracleAgent):
        def step(self):   # OracleAgent.step with the local solve above: process, scan, solve, update the duals
            self._process()
            self._scan()
            keys, idx, yl, yr = self.table()
            qi = None if self.qi is None else self.qi[idx]
            self.x, self.last_costs = arock_local_solve(self.x, self.fixed, self.ea, self.eb, self.split["rel"], self.split["sqrt_info"],
                                                        idx, qi, yr, self.rho_T, self.rho_theta, self.priors, cfg=lm_cfg)
            if keys:
                yl = pa.update_duals(yl, yr, pa.coords(self.x[idx], qi), self.eta)
                for k, key in enumerate(keys):
                    self.duals[key][0] = yl[k]
    return CeresLmAgent(split, **kw)
