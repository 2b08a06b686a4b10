"""Pose-graph side of libd2ba.so (include/d2pgo.h): ctypes binding, synthetic multi-agent pose graphs (BASELINE config 5:
10 000 poses on 8 random-walk trajectories, 40 000 edges), and g2o files in the reference's multi-agent convention.

g2o convention (d2pgo/test/posegraph_g2o.cpp:27-39, 57-232): `VERTEX_SE3:QUAT id x y z qx qy qz qw`,
`EDGE_SE3:QUAT id_a id_b x y z qx qy qz qw <21 upper-triangular information entries>`; for multi-agent files the top byte of
a vertex id carries chr('a' + agent) (gtsam Symbol style) and the low 56 bits the keyframe index.

4-DoF (d2pgo's default pgo_pose_dof = PGO_POSE_4D): `PgoSolver(pose_dof=4)` with set_poses_4d / add_edges_4d / get_poses_4d
on [x y z yaw] poses; poses_to_4d / poses_from_4d convert to and from 7-vector poses the way d2pgo does, pose_graph_to_4d
builds 4-DoF inputs from a make_pose_graph graph.

PCM (d2pgo's enable_pcm): `PgoSolver.pcm` rejects inconsistent loop closures before they are added (include/d2pgo.h
d2pgo_pcm); make_pcm_case builds its inputs from a make_pose_graph graph, with injected gross outliers.

Gravity prior (d2pgo's enable_gravity_prior, 6-DoF): `PgoSolver.add_gravity_priors` ties each pose's roll and pitch to the
gravity direction of its frame's ego (VIO) pose (include/d2pgo.h d2pgo_add_gravity_priors); make_gravity_case builds ego poses
for a make_pose_graph graph.

ARock (d2pgo's distributed pgo_mode 1): `ArockAgent` is one agent's handle in ARock mode (include/d2pgo.h d2pgo_arock_*);
arock_split builds agent s's sub-graph the way D2PGO::solve_multi does, arock_run runs the synchronous broadcast schedule.

Rotation initialisation (d2pgo's rotInitial, enable_rotation_initialization): `PgoSolver.rot_init` replaces the attitudes of the
free frames by d2pgo's chordal relaxation from the handle's edges and fixed frames (include/d2pgo.h d2pgo_rot_init), before
solve().  In ARock mode the distributed form (RotationInitARock): `ArockAgent.rot_init_step` / `rot_messages` / `rot_receive`
(include/d2pgo.h d2pgo_arock_rot_*), and arock_rot_init_run runs them on the synchronous schedule until rotInitial's
convergence gate, before arock_run.

Linear solver (the reference's ceres linear_solver_type): `PgoSolver(linear_solver="sparse_cholesky")` takes exact LM steps
from a GPU supernodal sparse Cholesky (d2pgo's SPARSE_NORMAL_CHOLESKY; include/d2pgo.h d2pgo_set_linear_solver) instead of the
default truncated block-Jacobi PCG ("pcg"); cholesky_stats() reports the factor's structure and timings, cholesky_symbolic() runs
the host analysis alone.

Minimiser (the reference's ceres minimizer_type and time budget): `PgoSolver.set_minimizer("ceres_lm", **cfg)` on a
sparse-Cholesky handle solves with ceres' Levenberg-Marquardt trust region as d2pgo runs it (include/d2pgo.h
d2pgo_set_minimizer; cfg overrides CeresLmConfig fields, e.g. max_solver_time_in_seconds), decided on the device in one graph
launch; minimizer_report() and debug_minimizer_trace() report the last solve.  "restated" is the default LM loop.

Perturbation chart (d2pgo's perturb_mode, every 6-DoF node): `PgoSolver.set_chart("perturb")` solves for the 6-vectors
[p, theta] with q = q_init (x) quatfromRotationVector(theta), kept across solves (include/d2pgo.h d2pgo_set_chart);
get_perturb / set_perturb read and write that state."""
import ctypes as C

import numpy as np

from .solver import lib as _lib


class PgoConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_iterations", C.c_int32), ("pcg_max_iterations", C.c_int32), ("pose_dof", C.c_int32),
                ("pcg_tolerance", C.c_double), ("lambda0", C.c_double), ("function_tolerance", C.c_double)]


class PgoReport(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("accepted", C.c_int32), ("pcg_iterations", C.c_int32), ("converged", C.c_int32),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("device_ms", C.c_double)]


class PcmConfig(C.Structure):
    _fields_ = [("pcm_thres", C.c_double), ("pos_covariance_per_meter", C.c_double), ("yaw_covariance_per_meter", C.c_double)]


class ArockConfig(C.Structure):
    _fields_ = [("self_id", C.c_int32), ("dual_state_init_to_zero", C.c_int32), ("rho_frame_T", C.c_double), ("rho_frame_theta", C.c_double),
                ("eta_k", C.c_double)]


class RotInitConfig(C.Structure):
    _fields_ = [("enable_gravity_prior", C.c_int32), ("pcg_max_iterations", C.c_int32), ("gravity_sqrt_info", C.c_double),
                ("pcg_tolerance", C.c_double)]


class RotInitReport(C.Structure):
    _fields_ = [("frames", C.c_int32), ("edges_used", C.c_int32), ("edges_dropped", C.c_int32), ("pcg_iterations", C.c_int32 * 3),
                ("residual", C.c_double * 3), ("state_changes", C.c_double), ("device_ms", C.c_double)]


class ArockRotInitConfig(C.Structure):
    _fields_ = [("enable_gravity_prior", C.c_int32), ("pcg_max_iterations", C.c_int32), ("gravity_sqrt_info", C.c_double),
                ("pcg_tolerance", C.c_double), ("rho_rot_mat", C.c_double)]


class CholeskyInfo(C.Structure):
    _fields_ = [("free_poses", C.c_int32), ("block_pairs", C.c_int32), ("nnz_L", C.c_int64), ("nnz_L_stored", C.c_int64),
                ("supernodes", C.c_int32), ("levels", C.c_int32), ("supernodes_fundamental", C.c_int32), ("levels_fundamental", C.c_int32),
                ("max_front_rows", C.c_int32), ("max_front_cols", C.c_int32), ("factorizations", C.c_int32),
                ("failed_factorizations", C.c_int32), ("factor_ms", C.c_double), ("solve_ms", C.c_double)]


LINEAR_SOLVERS = {"pcg": 0, "sparse_cholesky": 1}


class CeresLmConfig(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("max_num_consecutive_invalid_steps", C.c_int32), ("jacobi_scaling", C.c_int32),
                ("pad_", C.c_int32), ("max_solver_time_in_seconds", C.c_double), ("initial_trust_region_radius", C.c_double),
                ("max_trust_region_radius", C.c_double), ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double), ("function_tolerance", C.c_double),
                ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double)]


class MinimizerSummary(C.Structure):
    _fields_ = [("termination_type", C.c_int32), ("reason", C.c_int32), ("successful_steps", C.c_int32), ("unsuccessful_steps", C.c_int32),
                ("host_syncs", C.c_int32), ("pad_", C.c_int32), ("final_radius", C.c_double), ("elapsed_s", C.c_double),
                ("initial_cost", C.c_double), ("final_cost", C.c_double)]


class MinimizerIteration(C.Structure):
    _fields_ = [("cost", C.c_double), ("candidate_cost", C.c_double), ("model_cost_change", C.c_double), ("relative_decrease", C.c_double),
                ("step_norm", C.c_double), ("radius", C.c_double), ("decrease_factor", C.c_double), ("kind", C.c_int32), ("pad_", C.c_int32)]


MINIMIZERS = {"restated": 0, "ceres_lm": 1}
TERMINATIONS = {0: "CONVERGENCE", 1: "NO_CONVERGENCE", 2: "FAILURE"}
STOP_REASONS = {1: "gradient", 2: "parameter", 3: "function", 4: "min_radius", 5: "max_iterations", 6: "time", 7: "invalid_steps"}
STEP_KINDS = {0: "accepted", 1: "rejected", 2: "invalid", 3: "converged"}
TRACE_CAP = 16384   # trace records the library keeps per solve


def default_ceres_lm_config():
    """ceres' defaults as the library states them (d2pgo_default_ceres_lm_config), as a dict."""
    c = CeresLmConfig()
    _lib().d2pgo_default_ceres_lm_config(C.byref(c))
    return {k: getattr(c, k) for k, _ in CeresLmConfig._fields_ if k != "pad_"}


def _info_dict(r):
    return {k: getattr(r, k) for k, _ in CholeskyInfo._fields_}


def cholesky_symbolic(n, fixed, ea, eb, dof=6):
    """The sparse Cholesky's host analysis alone (no device, no handle; include/d2pgo.h d2pgo_cholesky_symbolic): n poses,
    fixed flags (None = all free), edge ends as pose indices, block size 4 or 6.  Returns dict(perm = pose of each block
    column [n_free], sn_ptr = first column of each supernode and the end, sn_parent, **the structure counts)."""
    f = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
    a = np.ascontiguousarray(ea, np.int32); b = np.ascontiguousarray(eb, np.int32)
    perm = np.zeros(max(n, 1), np.int32); ptr = np.zeros(n + 1, np.int32); par = np.zeros(max(n, 1), np.int32); info = CholeskyInfo()
    rc = _lib().d2pgo_cholesky_symbolic(C.c_int32(n), _p(f), C.c_int32(len(a)), _p(a), _p(b), C.c_int32(dof), _p(perm), _p(ptr), _p(par), C.byref(info))
    if rc:
        raise RuntimeError(f"d2pgo_cholesky_symbolic failed rc={rc}")
    S = info.supernodes
    return dict(perm=perm[: info.free_poses].copy(), sn_ptr=ptr[: S + 1].copy(), sn_parent=par[:S].copy(), **_info_dict(info))


class PcmReport(C.Structure):
    _fields_ = [("groups", C.c_int32), ("inliers", C.c_int32), ("pairs_tested", C.c_int64), ("consistent_pairs", C.c_int64),
                ("clique_rounds", C.c_int64), ("device_ms", C.c_double), ("pair_ms", C.c_double), ("clique_ms", C.c_double)]


class PcmStreamReport(C.Structure):
    _fields_ = [("new_loops", C.c_int32), ("total_loops", C.c_int32), ("groups", C.c_int32), ("groups_touched", C.c_int32), ("inliers", C.c_int32),
                ("pairs_tested", C.c_int64), ("consistent_pairs", C.c_int64), ("clique_rounds", C.c_int64), ("device_ms", C.c_double),
                ("pair_ms", C.c_double), ("clique_ms", C.c_double)]


PGO_EXPORTED = ["d2pgo_default_config", "d2pgo_create", "d2pgo_destroy", "d2pgo_last_error", "d2pgo_set_poses", "d2pgo_add_edges",
                "d2pgo_comm_init", "d2pgo_solve", "d2pgo_get_poses", "d2pgo_debug_edges", "d2pgo_set_poses_4d", "d2pgo_add_edges_4d",
                "d2pgo_get_poses_4d", "d2pgo_default_pcm_config", "d2pgo_pcm", "d2pgo_debug_pcm_smd", "d2pgo_debug_pcm_clique",
                "d2pgo_add_gravity_priors", "d2pgo_debug_gravity_priors", "d2pgo_default_arock_config", "d2pgo_arock_enable",
                "d2pgo_arock_receive", "d2pgo_arock_step", "d2pgo_arock_neighbours", "d2pgo_arock_duals", "d2pgo_debug_arock_terms",
                "d2pgo_default_rot_init_config", "d2pgo_rot_init", "d2pgo_set_linear_solver", "d2pgo_cholesky_stats",
                "d2pgo_debug_exact_step", "d2pgo_cholesky_symbolic", "d2pgo_debug_cholesky_system", "d2pgo_debug_pcg_step",
                "d2pgo_default_arock_rot_init_config", "d2pgo_arock_rot_init_step", "d2pgo_arock_rot_receive",
                "d2pgo_arock_rot_neighbours", "d2pgo_arock_rot_duals", "d2pgo_debug_arock_rot_state", "d2pgo_pcm_stream_reset",
                "d2pgo_pcm_stream", "d2pgo_debug_pcm_stream_smd", "d2pgo_debug_pcm_clique_inc",
                "d2pgo_default_ceres_lm_config", "d2pgo_set_minimizer", "d2pgo_minimizer_report", "d2pgo_debug_minimizer_trace",
                "d2pgo_set_chart", "d2pgo_set_perturb", "d2pgo_get_perturb"]
CHARTS = {"retraction": 0, "perturb": 1}
GRAVITY_SQRT_INFO = 10.0   # d2pgo's gravity_sqrt_info (RotInitConfig, d2pgo_config.h:13; the shipped configs)
_CREATE_ERRORS = {2: "pose_dof must be 0 or 6 (6-DoF poses) or 4 ([x y z yaw] poses)", 3: "no CUDA device (there is no CPU fallback)",
                  4: "bad device index"}


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class PgoSolver:
    def __init__(self, linear_solver="pcg", **kw):
        L = _lib()
        L.d2pgo_last_error.restype = C.c_char_p
        L.d2pgo_last_error.argtypes = [C.c_void_p]
        self.cfg = PgoConfig()
        L.d2pgo_default_config(C.byref(self.cfg))
        for k, v in kw.items():
            setattr(self.cfg, k, v)
        self.h = C.c_void_p()
        rc = L.d2pgo_create(C.byref(self.cfg), C.byref(self.h))
        if rc:
            raise RuntimeError(f"d2pgo_create failed rc={rc}: {_CREATE_ERRORS.get(rc, 'CUDA device required; no CPU fallback')}")
        self.n_poses = 0
        self.n_edges = 0
        self.n_priors = 0
        if linear_solver != "pcg":
            self.set_linear_solver(linear_solver)

    @property
    def dim(self):
        """The size D of a pose's tangent: 4 with pose_dof = 4, else 6."""
        return 4 if self.cfg.pose_dof == 4 else 6

    def set_linear_solver(self, kind):
        """"pcg" (the default) or "sparse_cholesky" (include/d2pgo.h d2pgo_set_linear_solver); ints pass through."""
        k = LINEAR_SOLVERS.get(kind, kind) if isinstance(kind, str) else int(kind)
        if isinstance(k, str):
            raise ValueError(f"unknown linear solver {kind!r}: {sorted(LINEAR_SOLVERS)}")
        self._chk(_lib().d2pgo_set_linear_solver(self.h, C.c_int32(k)), "set_linear_solver")

    def cholesky_stats(self):
        """Structure counts of the current graph's sparse Cholesky and the counters of the last solve, as a dict."""
        r = CholeskyInfo()
        self._chk(_lib().d2pgo_cholesky_stats(self.h, C.byref(r)), "cholesky_stats")
        return _info_dict(r)

    def debug_exact_step(self, lam):
        """The sparse Cholesky's step dx [N, D] for damping lam at the current poses (0 on fixed poses); poses unchanged."""
        out = np.zeros((self.n_poses, self.dim))
        self._chk(_lib().d2pgo_debug_exact_step(self.h, C.c_double(lam), _p(out), C.c_int64(out.size)), "debug_exact_step")
        return out

    def debug_pcg_step(self, lam, max_iterations, tolerance):
        """One PCG step (the default linear solver) for damping lam at the current poses, at most max_iterations iterations to
        relative residual tolerance: (dx [N, D] (0 on fixed poses), iterations run, the last relative residual); poses unchanged."""
        out = np.zeros((self.n_poses, self.dim)); it = C.c_int32(); res = C.c_double()
        self._chk(_lib().d2pgo_debug_pcg_step(self.h, C.c_double(lam), C.c_int32(max_iterations), C.c_double(tolerance), _p(out),
                                              C.c_int64(out.size), C.byref(it), C.byref(res)), "debug_pcg_step")
        return out, it.value, res.value

    def debug_cholesky_system(self):
        """The system the last sparse-Cholesky step on this handle factored, as the device assembled it (include/d2pgo.h
        d2pgo_debug_cholesky_system): dict(diag [N, D, D] damped diagonal blocks, b [N, D] = -g (both 0 on fixed poses),
        pairs [P, 2] pose indices a < b of each distinct free pair, pair_blocks [P, D, D] H_ab)."""
        D = self.dim
        P = self.cholesky_stats()["block_pairs"]
        diag = np.zeros((self.n_poses, D, D)); b = np.zeros((self.n_poses, D))
        ab = np.zeros((max(P, 1), 2), np.int32); H = np.zeros((max(P, 1), D, D)); n = C.c_int32()
        self._chk(_lib().d2pgo_debug_cholesky_system(self.h, _p(diag), _p(b), C.c_int32(P), C.byref(n), _p(ab), _p(H)), "debug_cholesky_system")
        return dict(diag=diag, b=b, pairs=ab[: n.value], pair_blocks=H[: n.value])

    def set_minimizer(self, kind, **cfg):
        """"restated" (the default LM loop) or "ceres_lm" (include/d2pgo.h d2pgo_set_minimizer): cfg overrides CeresLmConfig
        fields of ceres' defaults; ints pass through."""
        k = MINIMIZERS.get(kind, kind) if isinstance(kind, str) else int(kind)
        if isinstance(k, str):
            raise ValueError(f"unknown minimizer {kind!r}: {sorted(MINIMIZERS)}")
        c = CeresLmConfig()
        _lib().d2pgo_default_ceres_lm_config(C.byref(c))
        for name, v in cfg.items():
            if name not in dict(CeresLmConfig._fields_):
                raise KeyError(name)
            setattr(c, name, v)
        self._chk(_lib().d2pgo_set_minimizer(self.h, C.c_int32(k), C.byref(c)), "set_minimizer")

    def minimizer_report(self):
        """The ceres minimiser's report of the last solve or ARock step, as a dict (termination and reason as names)."""
        r = MinimizerSummary()
        self._chk(_lib().d2pgo_minimizer_report(self.h, C.byref(r)), "minimizer_report")
        out = {k: getattr(r, k) for k, _ in MinimizerSummary._fields_ if k != "pad_"}
        out["termination"] = TERMINATIONS.get(r.termination_type, r.termination_type)
        out["stop"] = STOP_REASONS.get(r.reason, r.reason)
        return out

    def debug_minimizer_trace(self):
        """Per iteration of the last ceres solve: dict of arrays cost, candidate_cost, model_cost_change, relative_decrease,
        step_norm, radius, decrease_factor (after the update) and kind (0 accepted, 1 rejected, 2 invalid, 3 converged)."""
        rep = self.minimizer_report()
        n_max = min(rep["successful_steps"] + rep["unsuccessful_steps"], TRACE_CAP)
        buf = (MinimizerIteration * max(n_max, 1))()
        n = C.c_int32()
        self._chk(_lib().d2pgo_debug_minimizer_trace(self.h, C.c_int32(n_max), C.byref(n), buf), "debug_minimizer_trace")
        names = [k for k, _ in MinimizerIteration._fields_ if k != "pad_"]
        return {k: np.array([getattr(buf[i], k) for i in range(n.value)], np.int32 if k == "kind" else np.float64) for k in names}

    def set_chart(self, chart, ids=None, q_init=None):
        """"perturb" solves in d2pgo's perturbation chart (include/d2pgo.h d2pgo_set_chart): every pose's state becomes [p, 0]
        with q_init its current attitude, or q_init [n, 4] (xyzw) for the listed ids; "retraction" (the default) leaves it."""
        k = CHARTS.get(chart, chart) if isinstance(chart, str) else int(chart)
        if isinstance(k, str):
            raise ValueError(f"unknown chart {chart!r}: {sorted(CHARTS)}")
        ids = np.zeros(0, np.int64) if ids is None else np.ascontiguousarray(ids, np.int64)
        q = None if q_init is None else np.ascontiguousarray(np.asarray(q_init, np.float64).reshape(-1, 4))
        self._chk(_lib().d2pgo_set_chart(self.h, C.c_int32(k), C.c_int32(len(ids)), _p(ids), _p(q)), "set_chart")

    def set_perturb(self, ids, x6):
        """The chart states [p, theta] of the listed poses."""
        ids = np.ascontiguousarray(ids, np.int64); x = np.ascontiguousarray(np.asarray(x6, np.float64).reshape(-1, 6))
        self._chk(_lib().d2pgo_set_perturb(self.h, C.c_int32(len(ids)), _p(ids), _p(x)), "set_perturb")

    def get_perturb(self, ids):
        """(x [n, 6] = [p, theta], q_init [n, 4]) of the listed poses of a chart handle."""
        ids = np.ascontiguousarray(ids, np.int64); x = np.zeros((len(ids), 6)); q = np.zeros((len(ids), 4))
        self._chk(_lib().d2pgo_get_perturb(self.h, C.c_int32(len(ids)), _p(ids), _p(x), _p(q)), "get_perturb")
        return x, q

    def _chk(self, rc, what):
        if rc:
            raise RuntimeError(f"{what} failed rc={rc}: {_lib().d2pgo_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            _lib().d2pgo_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_poses(self, ids, poses, fixed=None):
        ids = np.ascontiguousarray(ids, np.int64); poses = np.ascontiguousarray(poses, np.float64)
        f = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        self._chk(_lib().d2pgo_set_poses(self.h, C.c_int32(len(ids)), _p(ids), _p(poses), _p(f)), "set_poses")
        self.n_poses = len(ids)
        self.n_edges = 0
        self.n_priors = 0

    def add_edges(self, id_a, id_b, rel, sqrt_info):
        id_a = np.ascontiguousarray(id_a, np.int64); id_b = np.ascontiguousarray(id_b, np.int64)
        rel = np.ascontiguousarray(rel, np.float64); si = np.ascontiguousarray(sqrt_info, np.float64)
        self._chk(_lib().d2pgo_add_edges(self.h, C.c_int32(len(id_a)), _p(id_a), _p(id_b), _p(rel), _p(si)), "add_edges")
        self.n_edges += len(id_a)

    def set_poses_4d(self, ids, poses4, fixed=None):
        """[x y z yaw] poses of a pose_dof = 4 solver."""
        ids = np.ascontiguousarray(ids, np.int64); poses4 = np.ascontiguousarray(poses4, np.float64)
        f = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        self._chk(_lib().d2pgo_set_poses_4d(self.h, C.c_int32(len(ids)), _p(ids), _p(poses4), _p(f)), "set_poses_4d")
        self.n_poses = len(ids)
        self.n_edges = 0
        self.n_priors = 0

    def add_edges_4d(self, id_a, id_b, rel4, sqrt_info16):
        """rel4 = [x y z yaw] measurements (RelPoseFactor4D), sqrt_info16 = 4x4 square-root information per edge."""
        id_a = np.ascontiguousarray(id_a, np.int64); id_b = np.ascontiguousarray(id_b, np.int64)
        rel4 = np.ascontiguousarray(rel4, np.float64); si = np.ascontiguousarray(sqrt_info16, np.float64)
        self._chk(_lib().d2pgo_add_edges_4d(self.h, C.c_int32(len(id_a)), _p(id_a), _p(id_b), _p(rel4), _p(si)), "add_edges_4d")
        self.n_edges += len(id_a)

    def add_gravity_priors(self, ids, ego_poses7, sqrt_info=None):
        """One gravity prior per id (d2pgo's setupGravityPriorFactors): r = S^T (R_i^T e3 - R_ego^T e3) with the frame's ego pose
        [x y z qx qy qz qw]; sqrt_info = [n, 3, 3] (or [n, 9]) S, None = GRAVITY_SQRT_INFO * I3 for every prior.  6-DoF only."""
        ids = np.ascontiguousarray(ids, np.int64); ego = np.ascontiguousarray(np.asarray(ego_poses7, np.float64).reshape(-1, 7))
        S = np.tile(GRAVITY_SQRT_INFO * np.eye(3), (len(ids), 1, 1)) if sqrt_info is None else np.asarray(sqrt_info, np.float64)
        S = np.ascontiguousarray(S.reshape(-1, 9))
        self._chk(_lib().d2pgo_add_gravity_priors(self.h, C.c_int32(len(ids)), _p(ids), _p(ego), _p(S)), "add_gravity_priors")
        self.n_priors += len(ids)

    def debug_gravity_priors(self):
        """Per local gravity prior at the current poses: r (3) | J (3 x 6 in the tangent [dp, dtheta]), 21 doubles."""
        out = np.zeros((max(self.n_priors, 1), 21))
        self._chk(_lib().d2pgo_debug_gravity_priors(self.h, _p(out), C.c_int64(out.size)), "debug_gravity_priors")
        return out[: self.n_priors]

    def rot_init(self, ego_ids=None, ego_poses7=None, **cfg):
        """Chordal rotation initialisation (d2pgo's rotInitial; include/d2pgo.h d2pgo_rot_init): the attitudes of the free frames
        the edges name become the SO(3) projections of the linear least-squares rotations; positions, fixed frames and frames
        no edge names are kept.  cfg overrides RotInitConfig fields (enable_gravity_prior, pcg_max_iterations,
        gravity_sqrt_info, pcg_tolerance); with enable_gravity_prior every free frame an edge names needs an ego pose
        [x y z qx qy qz qw] in ego_ids / ego_poses7.  6-DoF only.  Returns the report as a dict."""
        return self._rot_init_call("rot_init", RotInitConfig(), _lib().d2pgo_default_rot_init_config, ego_ids, ego_poses7, cfg)

    def _rot_init_call(self, name, c, default, ego_ids, ego_poses7, cfg):
        """d2pgo_<name>(h, &c, n_ego, ego_ids, ego_poses7, &report), c filled by default(&c) and then cfg's overrides."""
        default(C.byref(c))
        for k, v in cfg.items():
            setattr(c, k, v)
        ids = np.zeros(0, np.int64) if ego_ids is None else np.ascontiguousarray(ego_ids, np.int64)
        ego = np.zeros((0, 7)) if ego_poses7 is None else np.ascontiguousarray(np.asarray(ego_poses7, np.float64).reshape(-1, 7))
        r = RotInitReport()
        self._chk(getattr(_lib(), f"d2pgo_{name}")(self.h, C.byref(c), C.c_int32(len(ids)), _p(ids), _p(ego), C.byref(r)), name)
        return _rot_report(r)

    def comm_init(self, unique_id, rank, nranks):
        uid = (C.c_uint8 * 128)(*unique_id)
        self._chk(_lib().d2pgo_comm_init(self.h, uid, C.c_int32(rank), C.c_int32(nranks)), "comm_init")

    def solve(self):
        r = PgoReport()
        self._chk(_lib().d2pgo_solve(self.h, C.byref(r)), "solve")
        return r

    def get_poses(self, ids):
        ids = np.ascontiguousarray(ids, np.int64); out = np.zeros((len(ids), 7))
        self._chk(_lib().d2pgo_get_poses(self.h, C.c_int32(len(ids)), _p(ids), _p(out)), "get_poses")
        return out

    def get_poses_4d(self, ids):
        ids = np.ascontiguousarray(ids, np.int64); out = np.zeros((len(ids), 4))
        self._chk(_lib().d2pgo_get_poses_4d(self.h, C.c_int32(len(ids)), _p(ids), _p(out)), "get_poses_4d")
        return out

    def debug_edges(self):
        """Per local edge: r | J_a | J_b at the current poses, 78 doubles (6-DoF) or 36 (pose_dof = 4)."""
        D = self.dim
        out = np.zeros((max(self.n_edges, 1), D + 2 * D * D))
        self._chk(_lib().d2pgo_debug_edges(self.h, _p(out), C.c_int64(out.size)), "debug_edges")
        return out[: self.n_edges]

    def pcm(self, frame_ids, frame_agent, ego_poses7, kf_a, kf_b, rel7, sqrt_info36, **cfg):
        """Loop-closure outlier rejection (d2pgo's enable_pcm; include/d2pgo.h d2pgo_pcm): boolean inlier mask over the loops.
        cfg overrides PcmConfig fields (pcm_thres, pos_covariance_per_meter, yaw_covariance_per_meter); the report of the
        call is kept in self.pcm_report.  The handle's poses and edges are not touched."""
        c = PcmConfig()
        _lib().d2pgo_default_pcm_config(C.byref(c))
        for k, v in cfg.items():
            setattr(c, k, v)
        fid = np.ascontiguousarray(frame_ids, np.int64); fag = np.ascontiguousarray(frame_agent, np.int32)
        ego = np.ascontiguousarray(ego_poses7, np.float64).reshape(-1, 7)
        ka = np.ascontiguousarray(kf_a, np.int64); kb = np.ascontiguousarray(kf_b, np.int64)
        rel = np.ascontiguousarray(rel7, np.float64).reshape(-1, 7); si = np.ascontiguousarray(sqrt_info36, np.float64).reshape(-1, 36)
        out = np.zeros(max(len(ka), 1), np.uint8); r = PcmReport()
        self._chk(_lib().d2pgo_pcm(self.h, C.byref(c), C.c_int32(len(fid)), _p(fid), _p(fag), _p(ego), C.c_int32(len(ka)), _p(ka), _p(kb), _p(rel), _p(si),
                                   _p(out), C.byref(r)), "pcm")
        self.pcm_report = r
        return out[: len(ka)].astype(bool)

    def debug_pcm_smd(self):
        """smd of every tested loop pair (i, j < i) of the last pcm() call, group-major (include/d2pgo.h)."""
        out = np.zeros(max(int(self.pcm_report.pairs_tested), 1))
        self._chk(_lib().d2pgo_debug_pcm_smd(self.h, _p(out), C.c_int64(out.size)), "debug_pcm_smd")
        return out[: int(self.pcm_report.pairs_tested)]

    # ---- PCM as a stream (include/d2pgo.h d2pgo_pcm_stream*)
    def pcm_stream_reset(self, incremental=0, **cfg):
        """Start a new PCM stream on this handle (forgets every frame, loop and clique); incremental 0 = maxCliqueHeu on the
        groups that get new loops, 1 = the incremental clique.  cfg overrides PcmConfig fields as for pcm()."""
        c = PcmConfig()
        _lib().d2pgo_default_pcm_config(C.byref(c))
        for k, v in cfg.items():
            setattr(c, k, v)
        self._chk(_lib().d2pgo_pcm_stream_reset(self.h, C.byref(c), C.c_int32(incremental)), "pcm_stream_reset")
        self.pcm_stream_report = None

    def pcm_stream(self, frame_ids, frame_agent, ego_poses7, loop_ids, kf_a, kf_b, rel7, sqrt_info36):
        """One call of the stream: the keyframes new since the last call, and the call's loops keyed by loop_ids (ids seen before
        are not tested again).  Boolean inlier mask over the call's loops; the report is kept in self.pcm_stream_report."""
        fid = np.ascontiguousarray(frame_ids, np.int64); fag = np.ascontiguousarray(frame_agent, np.int32)
        ego = np.ascontiguousarray(ego_poses7, np.float64).reshape(-1, 7)
        lid = np.ascontiguousarray(loop_ids, np.int64); ka = np.ascontiguousarray(kf_a, np.int64); kb = np.ascontiguousarray(kf_b, np.int64)
        rel = np.ascontiguousarray(rel7, np.float64).reshape(-1, 7); si = np.ascontiguousarray(sqrt_info36, np.float64).reshape(-1, 36)
        out = np.zeros(max(len(lid), 1), np.uint8); r = PcmStreamReport()
        self._chk(_lib().d2pgo_pcm_stream(self.h, C.c_int32(len(fid)), _p(fid), _p(fag), _p(ego), C.c_int32(len(lid)), _p(lid), _p(ka), _p(kb), _p(rel),
                                          _p(si), _p(out), C.byref(r)), "pcm_stream")
        self.pcm_stream_report = r
        return out[: len(lid)].astype(bool)

    def debug_pcm_stream_smd(self):
        """smd of the pairs tested by the last pcm_stream() call: groups in order of their first loop, new rows i ascending, j < i."""
        n = int(self.pcm_stream_report.pairs_tested)
        out = np.zeros(max(n, 1))
        self._chk(_lib().d2pgo_debug_pcm_stream_smd(self.h, _p(out), C.c_int64(out.size)), "debug_pcm_stream_smd")
        return out[:n]

    def debug_pcm_clique_inc(self, adj, n_new, prev_size):
        """The incremental clique kernel alone on a symmetric boolean adjacency [n, n] whose last n_new vertices are new ->
        (boolean membership [n] of the clique found, all False when no seed beats prev_size; FMC's return value)."""
        words = pcm_pack_bits(adj)
        n = len(words); member = np.zeros(max(n, 1), np.uint8); size = C.c_int32()
        self._chk(_lib().d2pgo_debug_pcm_clique_inc(self.h, C.c_int32(n), _p(words if n else np.zeros(1, np.uint32)), C.c_int32(n_new), C.c_int32(prev_size),
                                                    _p(member), C.byref(size)), "debug_pcm_clique_inc")
        return member[:n].astype(bool), size.value

    # ---- ARock (include/d2pgo.h d2pgo_arock_*)
    def arock_enable(self, ids, owner, q_init=None, **cfg):
        """ARock mode: owner agent per pose id, 6-DoF q_init [n, 4] (None = the attitudes given to set_poses); cfg overrides
        ArockConfig fields (self_id, dual_state_init_to_zero, rho_frame_T, rho_frame_theta, eta_k)."""
        c = ArockConfig()
        _lib().d2pgo_default_arock_config(C.byref(c))
        for k, v in cfg.items():
            setattr(c, k, v)
        ids = np.ascontiguousarray(ids, np.int64); own = np.ascontiguousarray(owner, np.int32)
        q = None if q_init is None else np.ascontiguousarray(np.asarray(q_init, np.float64).reshape(-1, 4))
        self._chk(_lib().d2pgo_arock_enable(self.h, C.byref(c), C.c_int32(len(ids)), _p(ids), _p(own), _p(q)), "arock_enable")
        self.arock_cfg = c

    def arock_receive(self, sender, target, frame_ids, duals, dim=None):
        f = np.ascontiguousarray(frame_ids, np.int64); d = np.ascontiguousarray(np.asarray(duals, np.float64).reshape(len(f), -1))
        self._chk(_lib().d2pgo_arock_receive(self.h, C.c_int32(sender), C.c_int32(target), C.c_int32(len(f)), _p(f),
                                             C.c_int32(d.shape[1] if dim is None else dim), _p(d)), "arock_receive")

    def arock_step(self):
        r = PgoReport()
        self._chk(_lib().d2pgo_arock_step(self.h, C.byref(r)), "arock_step")
        return r

    def arock_neighbours(self):
        n = C.c_int32()
        _lib().d2pgo_arock_neighbours(self.h, 0, C.byref(n), None)
        out = np.zeros(max(n.value, 1), np.int32)
        self._chk(_lib().d2pgo_arock_neighbours(self.h, C.c_int32(len(out)), C.byref(n), _p(out)), "arock_neighbours")
        return out[: n.value]

    def arock_duals(self, neighbour):
        """(frame ids, y_l [n, D], y_r [n, D]) of the duals held with `neighbour`, frame ids ascending."""
        n = C.c_int32()
        _lib().d2pgo_arock_duals(self.h, C.c_int32(neighbour), 0, C.byref(n), None, None, None)
        m = max(n.value, 1)
        f = np.zeros(m, np.int64); yl = np.zeros((m, self.dim)); yr = np.zeros((m, self.dim))
        self._chk(_lib().d2pgo_arock_duals(self.h, C.c_int32(neighbour), C.c_int32(m), C.byref(n), _p(f), _p(yl), _p(yr)), "arock_duals")
        return f[: n.value], yl[: n.value], yr[: n.value]

    def debug_arock_terms(self, n_duals):
        """Per dual in table order at the current poses: r (D) | J (D x D), D + D^2 doubles."""
        D = self.dim
        out = np.zeros((max(n_duals, 1), D + D * D))
        self._chk(_lib().d2pgo_debug_arock_terms(self.h, _p(out), C.c_int64(out.size)), "debug_arock_terms")
        return out[:n_duals]

    # ---- distributed rotation initialisation (include/d2pgo.h d2pgo_arock_rot_*)
    def arock_rot_init_step(self, ego_ids=None, ego_poses7=None, **cfg):
        """One RotationInitARock step on this ARock handle; cfg overrides ArockRotInitConfig fields (enable_gravity_prior,
        pcg_max_iterations, gravity_sqrt_info, pcg_tolerance, rho_rot_mat).  Returns the report as a dict."""
        return self._rot_init_call("arock_rot_init_step", ArockRotInitConfig(), _lib().d2pgo_default_arock_rot_init_config, ego_ids,
                                   ego_poses7, cfg)

    def arock_rot_receive(self, sender, target, frame_ids, duals, poses7, dim=9):
        f = np.ascontiguousarray(frame_ids, np.int64)
        d = np.ascontiguousarray(np.asarray(duals, np.float64).reshape(len(f), -1)); p = np.ascontiguousarray(np.asarray(poses7, np.float64).reshape(len(f), 7))
        self._chk(_lib().d2pgo_arock_rot_receive(self.h, C.c_int32(sender), C.c_int32(target), C.c_int32(len(f)), _p(f), C.c_int32(dim), _p(d), _p(p)),
                  "arock_rot_receive")

    def arock_rot_neighbours(self):
        n = C.c_int32()
        _lib().d2pgo_arock_rot_neighbours(self.h, 0, C.byref(n), None)
        out = np.zeros(max(n.value, 1), np.int32)
        self._chk(_lib().d2pgo_arock_rot_neighbours(self.h, C.c_int32(len(out)), C.byref(n), _p(out)), "arock_rot_neighbours")
        return out[: n.value]

    def arock_rot_duals(self, neighbour):
        """(frame ids ascending, y_l [n, 9], y_r [n, 9], this handle's poses [n, 7]) of the rotation duals held with `neighbour`."""
        n = C.c_int32()
        _lib().d2pgo_arock_rot_duals(self.h, C.c_int32(neighbour), 0, C.byref(n), None, None, None, None)
        m = max(n.value, 1)
        f = np.zeros(m, np.int64); yl = np.zeros((m, 9)); yr = np.zeros((m, 9)); ps = np.zeros((m, 7))
        self._chk(_lib().d2pgo_arock_rot_duals(self.h, C.c_int32(neighbour), C.c_int32(m), C.byref(n), _p(f), _p(yl), _p(yr), _p(ps)), "arock_rot_duals")
        return f[: n.value], yl[: n.value], yr[: n.value], ps[: n.value]

    def debug_arock_rot_state(self):
        """dict(state [N, 3, 3] R_state per pose (0 before its first step), flag [N] 0 unnamed / 1 free / 2 fixed, and the rotation
        dual table in table order: neighbour [K], frame [K], yl [K, 9], yr [K, 9])."""
        N = self.n_poses
        st = np.zeros((max(N, 1), 9)); fl = np.zeros(max(N, 1), np.uint8); n = C.c_int32()
        _lib().d2pgo_debug_arock_rot_state(self.h, _p(st), _p(fl), 0, C.byref(n), None, None, None, None)
        K = max(n.value, 1)
        nb = np.zeros(K, np.int32); fr = np.zeros(K, np.int64); yl = np.zeros((K, 9)); yr = np.zeros((K, 9))
        self._chk(_lib().d2pgo_debug_arock_rot_state(self.h, _p(st), _p(fl), C.c_int32(K), C.byref(n), _p(nb), _p(fr), _p(yl), _p(yr)),
                  "debug_arock_rot_state")
        k = n.value
        return dict(state=st[:N].reshape(N, 3, 3), flag=fl[:N].copy(), neighbour=nb[:k], frame=fr[:k], yl=yl[:k], yr=yr[:k])

    def debug_pcm_clique(self, adj):
        """The device clique kernel alone on a symmetric boolean adjacency [n, n] -> boolean membership [n]."""
        words = pcm_pack_bits(adj)
        n = len(words); member = np.zeros(max(n, 1), np.uint8); size = C.c_int32()
        self._chk(_lib().d2pgo_debug_pcm_clique(self.h, C.c_int32(n), _p(words), _p(member), C.byref(size)), "debug_pcm_clique")
        return member[:n].astype(bool)


def _rot_report(r):
    return dict(frames=r.frames, edges_used=r.edges_used, edges_dropped=r.edges_dropped, pcg_iterations=list(r.pcg_iterations),
                residual=list(r.residual), state_changes=r.state_changes, device_ms=r.device_ms)


def pcm_pack_bits(adj):
    """Boolean [n, n] -> uint32 rows [n, ceil(n / 32)], bit j of row i = word j // 32, bit j % 32 (d2pgo_debug_pcm_clique)."""
    adj = np.asarray(adj, bool); n = len(adj); W = (n + 31) // 32
    pad = np.zeros((n, W * 32), bool); pad[:, :n] = adj
    return np.ascontiguousarray((pad.reshape(n, W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32))


# ------------------------------------------------------------------------------------------------ synthetic graphs
def _qmul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def _qconj(q):
    return q * np.array([-1.0, -1.0, -1.0, 1.0])


def _qrot(q, v):
    qv = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], axis=-1)
    return _qmul(_qmul(q, qv), _qconj(q))[..., :3]


def _qexp(th):
    a = np.linalg.norm(th, axis=-1, keepdims=True)
    s = np.where(a < 1e-12, 0.5, np.sin(a / 2) / np.where(a < 1e-12, 1.0, a))
    return np.concatenate([th * s, np.cos(a / 2)], axis=-1)


def relative_pose(pa, pb):
    """T_a^-1 T_b as [t, q]."""
    qi = _qconj(pa[..., 3:7])
    return np.concatenate([_qrot(qi, pb[..., :3] - pa[..., :3]), _qmul(qi, pb[..., 3:7])], axis=-1)


def make_pose_graph(seed=0, n_agents=8, poses_per_agent=1250, loops=30000, sigma_t=0.05, sigma_r=np.deg2rad(1.0), loop_radius=5.0):
    """Random-walk trajectories (one per agent) + odometry edges + loop closures between poses within `loop_radius`
    (SURVEY.md 8d PGO config).  ids: agent * 1_000_000 + index.  Returns dict(ids, gt, init, fixed, id_a, id_b, rel, sqrt_info, agent)."""
    rng = np.random.default_rng(seed)
    gt = []
    for a in range(n_agents):
        p = np.zeros((poses_per_agent, 7)); p[0, :3] = rng.uniform(-10, 10, 3) * np.array([1, 1, 0.2]); p[0, 3:7] = _qexp(rng.normal(0, 0.3, 3) * np.array([0.2, 0.2, 3.0]))
        steps_t = np.abs(rng.normal(0.4, 0.1, (poses_per_agent, 1))) * np.array([1.0, 0.0, 0.0]) + rng.normal(0, 0.03, (poses_per_agent, 3))
        steps_r = rng.normal(0, 0.08, (poses_per_agent, 3)) * np.array([0.2, 0.2, 1.0])
        for k in range(1, poses_per_agent):
            p[k, :3] = p[k - 1, :3] + _qrot(p[k - 1, 3:7], steps_t[k]); q = _qmul(p[k - 1, 3:7], _qexp(steps_r[k])); p[k, 3:7] = q / np.linalg.norm(q)
        gt.append(p)
    gt = np.concatenate(gt); N = len(gt)
    agent = np.repeat(np.arange(n_agents), poses_per_agent)
    ids = (agent.astype(np.int64) * 1_000_000 + np.tile(np.arange(poses_per_agent), n_agents)).astype(np.int64)
    ia = [np.arange(a * poses_per_agent, (a + 1) * poses_per_agent - 1) for a in range(n_agents)]
    ia = np.concatenate(ia); ib = ia + 1
    # loop closures: random pairs within the radius (grid hashing)
    cell = np.floor(gt[:, :2] / loop_radius).astype(np.int64); key = cell[:, 0] * 100003 + cell[:, 1]
    order = np.argsort(key); ks = key[order]
    la, lb = [], []
    tries = 0
    while len(la) < loops and tries < 50:
        i = rng.integers(0, N, loops)
        lo = np.searchsorted(ks, key[i], "left"); hi = np.searchsorted(ks, key[i], "right")
        j = order[(lo + (rng.random(loops) * (hi - lo)).astype(np.int64)).clip(0, N - 1)]
        ok = (np.abs(i - j) > 5) & (np.linalg.norm(gt[i, :3] - gt[j, :3], axis=1) < loop_radius)
        la += i[ok].tolist(); lb += j[ok].tolist(); tries += 1
    la = la[:loops]; lb = lb[:loops]
    # one guaranteed inter-agent closure per agent (closest pair to any earlier agent) so that the graph is connected and the
    # single fixed pose removes the whole gauge freedom
    for a in range(1, n_agents):
        mine = np.arange(a * poses_per_agent, (a + 1) * poses_per_agent); prev = np.arange(0, a * poses_per_agent)
        sub = prev[:: max(1, len(prev) // 2000)]
        d2 = ((gt[mine, None, :3] - gt[None, sub, :3]) ** 2).sum(-1)
        i, j = np.unravel_index(np.argmin(d2), d2.shape)
        la.append(int(mine[i])); lb.append(int(sub[j]))
    la = np.array(la, np.int64); lb = np.array(lb, np.int64)
    ea = np.concatenate([ia, la]); eb = np.concatenate([ib, lb]); E = len(ea)
    rel = relative_pose(gt[ea], gt[eb])
    rel[:, :3] += rng.normal(0, sigma_t, (E, 3))
    q = _qmul(rel[:, 3:7], _qexp(rng.normal(0, sigma_r, (E, 3)))); rel[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    si = np.zeros((E, 6, 6)); si[:, [0, 1, 2], [0, 1, 2]] = 1.0 / sigma_t; si[:, [3, 4, 5], [3, 4, 5]] = 1.0 / sigma_r
    # initial guess: odometry chained per agent (drifts), first pose of every agent from ground truth + noise
    init = gt.copy()
    for a in range(n_agents):
        s = a * poses_per_agent
        init[s, :3] += rng.normal(0, 0.2, 3)
        for k in range(1, poses_per_agent):
            r = rel[s - a + k - 1] if False else rel[(s - a) + k - 1]   # odometry edge index of (s+k-1 -> s+k)
            init[s + k, :3] = init[s + k - 1, :3] + _qrot(init[s + k - 1, 3:7], r[:3]); q = _qmul(init[s + k - 1, 3:7], r[3:7]); init[s + k, 3:7] = q / np.linalg.norm(q)
    fixed = np.zeros(N, np.uint8); fixed[0] = 1; init[0] = gt[0]
    return dict(ids=ids, gt=gt, init=init, fixed=fixed, id_a=ids[ea], id_b=ids[eb], rel=rel, sqrt_info=si.reshape(E, 36), agent=agent, ea=ea, eb=eb)


# ------------------------------------------------------------------------------------------------ 4-DoF poses
def normalize_angle(a):
    """Utility::NormalizeAngle (utils.hpp:251-257): a - 2 pi floor((a + pi) / 2 pi), in [-pi, pi)."""
    return a - 2.0 * np.pi * np.floor((a + np.pi) / (2.0 * np.pi))


def quat_yaw(q):
    """Yaw of [qx qy qz qw] quaternions: the z angle of the z-y-x Euler decomposition, atan2(2(w z + x y), 1 - 2(y^2 + z^2)).
    ASSUMED to be Swarm::Pose::yaw (swarm_msgs is not in the reference tree); the same formula pins RelPoseFactor4D's
    measurement yaw to the reference functor."""
    q = np.asarray(q, np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))


def _qyaw(yaw):
    yaw = np.asarray(yaw, np.float64)
    z = np.zeros_like(yaw)
    return np.stack([z, z, np.sin(yaw / 2), np.cos(yaw / 2)], axis=-1)


def poses_to_4d(poses7):
    """[x y z qx qy qz qw] -> [x y z yaw], as PGOState::addFrame's 4-DoF branch takes a frame (pgostate.hpp:31-33,
    Swarm::Pose::to_vector_xyzyaw; yaw by quat_yaw, the ASSUMED Swarm::Pose::yaw)."""
    p = np.asarray(poses7, np.float64)
    return np.concatenate([p[..., :3], quat_yaw(p[..., 3:7])[..., None]], axis=-1)


def poses_from_4d(x4, ego_poses7):
    """Solved [x y z yaw] -> [x y z qx qy qz qw] with the ego pose's roll and pitch put back, as D2PGO::getOptimizedTrajs does
    for 4-DoF (d2pgo.cpp:640-645): q = Rz(yaw) (yaw_only(q_ego)^-1 q_ego)."""
    x4 = np.asarray(x4, np.float64); qe = np.asarray(ego_poses7, np.float64)[..., 3:7]
    tilt = _qmul(_qconj(_qyaw(quat_yaw(qe))), qe)
    q = _qmul(_qyaw(x4[..., 3]), tilt)
    return np.concatenate([x4[..., :3], q / np.linalg.norm(q, axis=-1, keepdims=True)], axis=-1)


def pose_graph_to_4d(g, seed=0, sigma_t=0.05, sigma_yaw=np.deg2rad(1.0)):
    """4-DoF inputs from a make_pose_graph graph: the same ground truth (as [x y z yaw]) and the same edge topology, measurements
    Rz(-yaw_a)(p_b - p_a) + noise and N(yaw_b - yaw_a + noise), diagonal square-root information, initial guess chained from the
    odometry edges per agent (first pose of every agent from ground truth + noise), pose 0 fixed at ground truth.
    Returns dict(ids, gt, init, fixed, id_a, id_b, ea, eb, rel, sqrt_info, agent) with 4-vectors and [E, 16] sqrt_info."""
    rng = np.random.default_rng(seed)
    gt = poses_to_4d(g["gt"]); ea = np.asarray(g["ea"]); eb = np.asarray(g["eb"]); agent = np.asarray(g["agent"])
    E = len(ea)
    c, s = np.cos(-gt[ea, 3]), np.sin(-gt[ea, 3]); v = gt[eb, :3] - gt[ea, :3]
    rel = np.zeros((E, 4))
    rel[:, 0] = c * v[:, 0] - s * v[:, 1] + rng.normal(0, sigma_t, E)
    rel[:, 1] = s * v[:, 0] + c * v[:, 1] + rng.normal(0, sigma_t, E)
    rel[:, 2] = v[:, 2] + rng.normal(0, sigma_t, E)
    rel[:, 3] = normalize_angle(gt[eb, 3] - gt[ea, 3] + rng.normal(0, sigma_yaw, E))
    si = np.zeros((E, 4, 4)); si[:, [0, 1, 2], [0, 1, 2]] = 1.0 / sigma_t; si[:, 3, 3] = 1.0 / sigma_yaw
    # odometry edges: e -> (i, i + 1) within one agent; each pose after an agent's first has exactly one (make_pose_graph lists
    # them first)
    odo = np.full(len(gt), -1)
    n_odo = len(gt) - len(np.unique(agent))
    assert np.all(eb[:n_odo] == ea[:n_odo] + 1) and np.all(agent[ea[:n_odo]] == agent[eb[:n_odo]])
    odo[eb[:n_odo]] = np.arange(n_odo)
    init = gt.copy()
    for a in np.unique(agent):
        idx = np.nonzero(agent == a)[0]; s0 = idx[0]
        e = odo[idx[1:]]
        assert np.all(e >= 0)
        init[s0, :3] += rng.normal(0, 0.2, 3)
        yaw = init[s0, 3] + np.concatenate([[0.0], np.cumsum(rel[e, 3])])
        c, s = np.cos(yaw[:-1]), np.sin(yaw[:-1])
        step = np.stack([c * rel[e, 0] - s * rel[e, 1], s * rel[e, 0] + c * rel[e, 1], rel[e, 2]], axis=1)
        init[idx, :3] = init[s0, :3] + np.concatenate([np.zeros((1, 3)), np.cumsum(step, axis=0)])
        init[idx, 3] = normalize_angle(yaw)
    fixed = np.zeros(len(gt), np.uint8); fixed[0] = 1; init[0] = gt[0]
    return dict(ids=np.asarray(g["ids"]), gt=gt, init=init, fixed=fixed, id_a=np.asarray(g["id_a"]), id_b=np.asarray(g["id_b"]), ea=ea, eb=eb,
                rel=rel, sqrt_info=si.reshape(E, 16), agent=agent)


# ------------------------------------------------------------------------------------------------ PCM cases
def _odometry_chain(g):
    """Per-agent ego trajectories: the first pose of every agent from ground truth, then the odometry edges composed."""
    gt = np.asarray(g["gt"]); agent = np.asarray(g["agent"]); ea = np.asarray(g["ea"]); eb = np.asarray(g["eb"]); rel = np.asarray(g["rel"])
    n_odo = len(gt) - len(np.unique(agent))
    assert np.all(eb[:n_odo] == ea[:n_odo] + 1)
    ego = gt.copy()
    for e in range(n_odo):
        a, b = ea[e], eb[e]
        ego[b, :3] = ego[a, :3] + _qrot(ego[a, 3:7], rel[e, :3]); q = _qmul(ego[a, 3:7], rel[e, 3:7]); ego[b, 3:7] = q / np.linalg.norm(q)
    return ego, n_odo


def make_pcm_case(g, outlier_frac=0.05, seed=0):
    """A PCM input from a make_pose_graph graph: frames = every pose with its agent and its ego pose (the agent's odometry
    chain), loops = the edges after the odometry edges, `rel_bad` = the same loops with a fraction turned into gross
    outliers (2-10 m of translation in a random direction and 20-180 degrees of yaw, random sign), `outlier` = which,
    `bad_dt` / `bad_yaw` = the perturbations of the outliers in loop order (to corrupt 4-DoF measurements the same way)."""
    rng = np.random.default_rng(seed)
    ego, n_odo = _odometry_chain(g)
    ids = np.asarray(g["ids"]); agent = np.asarray(g["agent"]).astype(np.int32)
    rel = np.array(g["rel"][n_odo:]); L = len(rel)
    bad = np.zeros(L, bool); bad[rng.choice(L, int(round(outlier_frac * L)), replace=False)] = True
    k = int(bad.sum())
    d = rng.normal(size=(k, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rel_bad = rel.copy()
    rel_bad[bad, :3] += d * rng.uniform(2.0, 10.0, (k, 1))
    yaw = rng.uniform(np.deg2rad(20), np.pi, k) * rng.choice([-1.0, 1.0], k)
    q = _qmul(rel_bad[bad, 3:7], _qyaw(yaw)); rel_bad[bad, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return dict(frame_ids=ids, frame_agent=agent, ego=ego, kf_a=np.asarray(g["id_a"][n_odo:]), kf_b=np.asarray(g["id_b"][n_odo:]), rel=rel,
                rel_bad=rel_bad, sqrt_info=np.asarray(g["sqrt_info"][n_odo:]), outlier=bad, bad_dt=d * np.linalg.norm(rel_bad[bad, :3] - rel[bad, :3], axis=1, keepdims=True),
                bad_yaw=yaw, n_odo=n_odo)


def pcm_arrival_steps(case, n_steps):
    """Splits a make_pcm_case input into arrival batches, as a PCM stream would receive it: each drone's keyframes are revealed
    in trajectory order, spread evenly over n_steps steps, and a loop arrives in the first step in which both its keyframes
    exist (loops of one step in input order).  -> list of (frame indices, loop indices) per step; steps may be empty."""
    agent = np.asarray(case["frame_agent"])
    step = np.zeros(len(agent), np.int64)
    for a in np.unique(agent):
        f = np.nonzero(agent == a)[0]
        step[f] = np.arange(len(f)) * n_steps // len(f)
    fidx = {int(f): k for k, f in enumerate(np.asarray(case["frame_ids"]).tolist())}
    la = np.array([fidx[int(k)] for k in np.asarray(case["kf_a"])], np.int64); lb = np.array([fidx[int(k)] for k in np.asarray(case["kf_b"])], np.int64)
    lstep = np.maximum(step[la], step[lb]) if len(la) else np.zeros(0, np.int64)
    return [(np.nonzero(step == t)[0], np.nonzero(lstep == t)[0]) for t in range(n_steps)]


def pcm_stream_args(case, frames, loops, rel_key="rel_bad"):
    """The arguments of PgoSolver.pcm_stream for frame and loop indices of a make_pcm_case input (loop id = its index)."""
    return (np.asarray(case["frame_ids"])[frames], np.asarray(case["frame_agent"])[frames], np.asarray(case["ego"])[frames], np.asarray(loops, np.int64),
            np.asarray(case["kf_a"])[loops], np.asarray(case["kf_b"])[loops], np.asarray(case[rel_key])[loops],
            np.asarray(case["sqrt_info"]).reshape(-1, 36)[loops])


# ------------------------------------------------------------------------------------------------ gravity priors
def make_gravity_case(g, sigma_tilt=np.deg2rad(0.5), seed=0):
    """Ego (VIO) poses for gravity priors on a make_pose_graph graph: position and yaw from the agent's odometry chain
    (_odometry_chain), roll and pitch from the ground truth turned by a random rotation of sigma_tilt per axis -- the gravity
    direction a VIO front end observes.  The graph's own odometry drifts in roll and pitch, which the priors correct.
    Returns dict(ids, ego) with ego [N, 7]."""
    rng = np.random.default_rng(seed)
    chain, _ = _odometry_chain(g)
    gt = np.asarray(g["gt"])
    tilt = _qmul(_qconj(_qyaw(quat_yaw(gt[:, 3:7]))), gt[:, 3:7])                 # ground-truth roll and pitch (zero yaw)
    tilt = _qmul(tilt, _qexp(rng.normal(0.0, sigma_tilt, (len(gt), 3))))
    q = _qmul(_qyaw(quat_yaw(chain[:, 3:7])), tilt)
    ego = np.concatenate([chain[:, :3], q / np.linalg.norm(q, axis=1, keepdims=True)], axis=1)
    return dict(ids=np.asarray(g["ids"]), ego=ego)


# ------------------------------------------------------------------------------------------------ g2o files
_IDX_AGENT_MIN = 1 << 56


def g2o_vertex_id(agent, index, multi=True):
    return (int(ord("a") + agent) << 56) | int(index) if multi else int(index)


def g2o_split_id(v):
    """posegraph_g2o.cpp:27-39 extrackKeyframeId: (agent, keyframe index)."""
    v = int(v)
    if v < _IDX_AGENT_MIN:
        return 0, v
    return ((v >> 56) & 255) - 97, v & ((1 << 56) - 1)


def write_g2o(path, ids, poses, id_a, id_b, rel, sqrt_info, multi=True):
    def vid(i):
        return g2o_vertex_id(int(i) // 1_000_000, int(i) % 1_000_000, multi)
    with open(path, "w") as f:
        for i, p in zip(ids, poses):
            f.write("VERTEX_SE3:QUAT %d %s\n" % (vid(i), " ".join(repr(float(x)) for x in p)))
        for a, b, r, s in zip(id_a, id_b, rel, np.asarray(sqrt_info).reshape(-1, 6, 6)):
            info = s.T @ s
            up = [info[i, j] for i in range(6) for j in range(i, 6)]
            f.write("EDGE_SE3:QUAT %d %d %s %s\n" % (vid(a), vid(b), " ".join(repr(float(x)) for x in r), " ".join(repr(float(x)) for x in up)))


def read_g2o(path, max_agent_id=1000):
    """-> dict(ids, poses, id_a, id_b, rel, sqrt_info); ids = agent * 1_000_000 + keyframe index (the estimator's frame-id
    convention, d2frontend_types.h:10-14).  Edges touching an agent above max_agent_id are skipped like the reference reader."""
    ids, poses, ea, eb, rel, si = [], [], [], [], [], []
    for line in open(path):
        t = line.split()
        if not t:
            continue
        if t[0] == "VERTEX_SE3:QUAT":
            ag, k = g2o_split_id(t[1])
            if ag > max_agent_id:
                continue
            p = np.array(t[2:9], float); p[3:7] /= np.linalg.norm(p[3:7])
            ids.append(ag * 1_000_000 + k); poses.append(p)
        elif t[0] == "EDGE_SE3:QUAT":
            (aa, ka), (ab, kb) = g2o_split_id(t[1]), g2o_split_id(t[2])
            if aa > max_agent_id or ab > max_agent_id:
                continue
            r = np.array(t[3:10], float); r[3:7] /= np.linalg.norm(r[3:7])
            up = np.array(t[10:31], float); info = np.zeros((6, 6)); k = 0
            for i in range(6):
                for j in range(i, 6):
                    info[i, j] = info[j, i] = up[k]; k += 1
            ea.append(aa * 1_000_000 + ka); eb.append(ab * 1_000_000 + kb); rel.append(r)
            w, V = np.linalg.eigh(info)           # symmetric square root of the information matrix
            si.append((V * np.sqrt(np.maximum(w, 0.0))) @ V.T)
    return dict(ids=np.array(ids, np.int64), poses=np.array(poses), id_a=np.array(ea, np.int64), id_b=np.array(eb, np.int64),
                rel=np.array(rel), sqrt_info=np.array(si).reshape(-1, 36))


def write_g2o_agents(directory, ids, poses, id_a, id_b, rel, sqrt_info):
    """The reference's multi-agent layout (read_g2o_multi_agents, posegraph_g2o.cpp:177-195): one file `<agent>.g2o` per
    agent with that agent's vertices and the edges that start at one of them (inter-agent edges name the other agent through the
    agent byte of the vertex id)."""
    import os
    ids = np.asarray(ids); id_a = np.asarray(id_a)
    agents = sorted(set(int(i) // 1_000_000 for i in ids))
    for a in agents:
        v = (ids // 1_000_000) == a; e = (id_a // 1_000_000) == a
        write_g2o(os.path.join(directory, f"{a}.g2o"), ids[v], np.asarray(poses)[v], id_a[e], np.asarray(id_b)[e], np.asarray(rel)[e], np.asarray(sqrt_info).reshape(-1, 36)[e])
    return agents


def read_g2o_agents(directory, agents_num):
    """Mirror of read_g2o_multi_agents: the numerically named *.g2o files in ascending order, the first `agents_num` of them,
    vertices / edges of agents above agents_num - 1 dropped; concatenated into one graph."""
    import os
    files = sorted((int(f[:-4]), os.path.join(directory, f)) for f in os.listdir(directory) if f.endswith(".g2o") and f[:-4].isdigit())[:agents_num]
    parts = [read_g2o(p, max_agent_id=agents_num - 1) for _, p in files]
    cat = lambda k: np.concatenate([q[k] for q in parts]) if parts else np.zeros(0)
    return dict(ids=cat("ids"), poses=cat("poses"), id_a=cat("id_a"), id_b=cat("id_b"), rel=cat("rel"), sqrt_info=cat("sqrt_info"))


# ------------------------------------------------------------------------------------------------ ARock (pgo_mode 1)
def graph_agents(g):
    """Owner agent of every pose of a graph dict: g["agent"], or the estimator's frame-id convention id // 1_000_000."""
    return np.asarray(g["agent"]) if "agent" in g else (np.asarray(g["ids"]) // 1_000_000).astype(np.int64)


def arock_split(g, s, main_id=0):
    """Agent s's sub-graph as D2PGO::solve_multi builds it: s's own ego-motion edges (setupEgoMotionFactors(solver, self_id),
    d2pgo.cpp:561-567) and every loop whose two frames s knows (setupLoopFactors, :413-466), where s knows its own frames and
    the frames at the other end of its loops.  An ego-motion edge joins two consecutive frames (in id order) of one agent;
    every other edge is a loop.  Only main_id's head frame is fixed, and only in main_id's own sub-graph (d2pgo.cpp:602-612).
    g: dict(ids, init or poses, id_a, id_b, rel, sqrt_info[, agent]) with 7-vector (6-DoF) or 4-vector (4-DoF) poses, e.g.
    from make_pose_graph, pose_graph_to_4d or read_g2o_agents.  Returns dict(self_id, ids, poses, fixed, owner, id_a, id_b,
    rel, sqrt_info, edges) with the frames in id order and `edges` the indices of the kept edges in g."""
    ids = np.asarray(g["ids"]); poses = np.asarray(g["init"] if "init" in g else g["poses"]); agent = graph_agents(g)
    pos = {int(i): k for k, i in enumerate(ids)}
    ia = np.array([pos[int(i)] for i in g["id_a"]], np.int64); ib = np.array([pos[int(i)] for i in g["id_b"]], np.int64)
    # consecutive frames of each agent, in id order
    nxt = {}
    for a in np.unique(agent):
        mine = np.sort(ids[agent == a])
        nxt.update({int(u): int(v) for u, v in zip(mine[:-1], mine[1:])})
    ida, idb = ids[ia], ids[ib]
    ego = np.array([(agent[x] == agent[y]) and (nxt.get(int(u)) == int(v) or nxt.get(int(v)) == int(u)) for x, y, u, v in zip(ia, ib, ida, idb)], bool)
    own = agent[ia] == s
    known = set(ids[agent == s].tolist())
    touch = ~ego & ((agent[ia] == s) | (agent[ib] == s))
    known |= set(ida[touch].tolist()) | set(idb[touch].tolist())
    kin = np.array([int(u) in known and int(v) in known for u, v in zip(ida, idb)], bool)
    keep = np.nonzero((ego & own) | (~ego & kin))[0]
    used = np.unique(np.concatenate([ia[keep], ib[keep]])) if len(keep) else np.zeros(0, np.int64)
    used = used[np.argsort(ids[used], kind="stable")]
    fixed = np.zeros(len(used), np.uint8)
    if s == main_id:
        head = ids[agent == s].min()
        fixed[ids[used] == head] = 1
    return dict(self_id=int(s), ids=ids[used].astype(np.int64), poses=poses[used].copy(), fixed=fixed, owner=agent[used].astype(np.int32),
                id_a=ida[keep].astype(np.int64), id_b=idb[keep].astype(np.int64), rel=np.asarray(g["rel"])[keep], sqrt_info=np.asarray(g["sqrt_info"])[keep], edges=keep)


class ArockAgent:
    """One agent of d2pgo's ARock mode on the GPU: a PgoSolver handle with the agent's sub-graph (arock_split) in ARock mode.
    q_init: 6-DoF attitudes [n, 4] of the sub-graph's frames (None = their initial attitudes); ego_poses: 6-DoF ego poses [n, 7]
    of the frames for one gravity prior each (d2pgo's enable_gravity_prior; None = no priors); cfg: ArockConfig fields;
    solver_kw: PgoConfig fields (pose_dof is taken from the poses)."""

    def __init__(self, split, q_init=None, ego_poses=None, solver_kw=None, **cfg):
        self.split = split; self.self_id = split["self_id"]; self.ego_poses = ego_poses
        self.dof = 4 if np.asarray(split["poses"]).shape[1] == 4 else 6
        self.s = PgoSolver(pose_dof=self.dof, **(solver_kw or {}))
        if self.dof == 4:
            self.s.set_poses_4d(split["ids"], split["poses"], split["fixed"]); self.s.add_edges_4d(split["id_a"], split["id_b"], split["rel"], split["sqrt_info"])
        else:
            self.s.set_poses(split["ids"], split["poses"], split["fixed"]); self.s.add_edges(split["id_a"], split["id_b"], split["rel"], split["sqrt_info"])
            if ego_poses is not None:
                self.s.add_gravity_priors(split["ids"], ego_poses)
        self.s.arock_enable(split["ids"], split["owner"], q_init, self_id=self.self_id, **cfg)

    def step(self):
        return self.s.arock_step()

    def messages(self):
        """broadcastData: one (sender, target, frame ids, y_l) per neighbour, neighbours ascending."""
        return [(self.self_id, int(n), *self.s.arock_duals(int(n))[:2]) for n in self.s.arock_neighbours()]

    def receive(self, msg):
        sender, target, frames, duals = msg
        self.s.arock_receive(sender, target, frames, duals)

    def duals(self):
        """{(neighbour, frame id): (y_l, y_r)}"""
        out = {}
        for n in self.s.arock_neighbours():
            f, yl, yr = self.s.arock_duals(int(n))
            out.update({(int(n), int(i)): (a, b) for i, a, b in zip(f, yl, yr)})
        return out

    def poses(self):
        ids = self.split["ids"]
        return self.s.get_poses_4d(ids) if self.dof == 4 else self.s.get_poses(ids)

    def rot_init_step(self, ego_poses7=None, **cfg):
        """One distributed rotation-initialisation step (RotationInitARock; PgoSolver.arock_rot_init_step); 6-DoF only.
        ego_poses7 [n, 7]: the ego poses of the sub-graph's frames for the gravity rows (None = the agent's ego_poses)."""
        ego = self.ego_poses if ego_poses7 is None else ego_poses7
        return self.s.arock_rot_init_step(None if ego is None else self.split["ids"], ego, **cfg)

    def rot_messages(self):
        """The rotation-initialisation broadcast: one (sender, target, frame ids, y_l [n, 9], poses [n, 7]) per neighbour."""
        out = []
        for n in self.s.arock_rot_neighbours():
            f, yl, _, ps = self.s.arock_rot_duals(int(n))
            out.append((self.self_id, int(n), f, yl, ps))
        return out

    def rot_receive(self, msg):
        sender, target, frames, duals, poses = msg
        self.s.arock_rot_receive(sender, target, frames, duals, poses)

    def close(self):
        self.s.close()


def arock_run(agents, rounds, after_round=None):
    """The synchronous broadcast schedule: every round, every agent steps, then every message of the round is delivered to every
    other agent (in the order of the agents, each agent's messages by neighbour).  after_round(r, agents, reports) is called
    after each round's delivery.  Returns the per-round lists of step reports."""
    out = []
    for r in range(rounds):
        reps = [a.step() for a in agents]
        msgs = [m for a in agents for m in a.messages()]
        for a in agents:
            for m in msgs:
                if m[0] != a.self_id:
                    a.receive(m)
        out.append(reps)
        if after_round is not None:
            after_round(r, agents, reps)
    return out


def rot_init_converged(state_changes, rounds_run, eps=1e-2, min_rounds=10):
    """D2PGO::rotInitial's gate (d2pgo.cpp:351-353): state_changes < eps with more than min_rounds solves before this one."""
    return state_changes < eps and rounds_run - 1 > min_rounds


def arock_rot_init_run(agents, max_rounds, eps=1e-2, min_rounds=10, after_round=None, **cfg):
    """d2pgo's distributed rotation initialisation on the synchronous schedule of arock_run: every round, every agent that has
    not converged steps (agent.rot_init_step(**cfg)), then every message of the round goes to every other agent.  An agent
    stops stepping and broadcasting once rot_init_converged holds for its report (rotInitial's is_rot_init_convergence) but
    keeps receiving.  after_round(r, agents, reports) after each round's delivery (None for an
    agent that did not step).  Returns the 1-based round at which each agent converged, None where it did not within
    max_rounds."""
    done = [None] * len(agents)
    for r in range(max_rounds):
        reps = []
        for i, a in enumerate(agents):
            if done[i] is not None:
                reps.append(None); continue
            rep = a.rot_init_step(**cfg)
            reps.append(rep)
            if rot_init_converged(rep["state_changes"], r + 1, eps, min_rounds):
                done[i] = r + 1
        msgs = [m for a, rep in zip(agents, reps) if rep is not None for m in a.rot_messages()]
        for a in agents:
            for m in msgs:
                if m[0] != a.self_id:
                    a.rot_receive(m)
        if after_round is not None:
            after_round(r, agents, reps)
        if all(d is not None for d in done):
            break
    return done
