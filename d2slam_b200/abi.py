"""ctypes / numpy mirrors of the C ABI declared in include/d2ba.h.

Only layout definitions live here (no compute).  The numpy dtypes are byte-compatible with
the C structs so arrays built by the synthetic harness can be handed to ``libd2ba.so``
(and, in tests only, to the CPU oracle) without copies.
"""
import ctypes as C

import numpy as np

D2BA_VERSION = 1

# d2ba_block_kind (reference ParamsType, d2common/include/d2common/solver/BaseParamResInfo.hpp:7-17)
POSE, EXTRINSIC, SPEED_BIAS, TD, LANDMARK = 0, 1, 2, 3, 4
KIND_SIZE = {POSE: 7, EXTRINSIC: 7, SPEED_BIAS: 9, TD: 1, LANDMARK: 1}
KIND_EFF = {POSE: 6, EXTRINSIC: 6, SPEED_BIAS: 9, TD: 1, LANDMARK: 1}

# d2ba_proj_type
PROJ_2F1C, PROJ_2F2C, PROJ_1F2C, PROJ_2F1C_DEPTH, PROJ_DEPTH_PRIOR = 0, 1, 2, 3, 4

TERM_NO_CONVERGENCE, TERM_FUNCTION_TOL, TERM_GRADIENT_TOL, TERM_PARAMETER_TOL, TERM_FAILURE = range(5)

# d2ba_debug_item
(DBG_N_CAM, DBG_HCC, DBG_GC, DBG_HLL, DBG_GL, DBG_W, DBG_COST, DBG_S, DBG_N_LC, DBG_OBS_INDEX,
 DBG_COL_OF_BLOCK, DBG_PROJ_RESJAC, DBG_STEP, DBG_GN_STEP, DBG_IMU_RESJAC, DBG_CONS_RESJAC, DBG_SOLVE_PATH, DBG_PLAN,
 DBG_LIN_JOBS) = range(19)
# the int64 fields of DBG_PLAN, in order
PLAN_FIELDS = ("fused_solve", "schur_small", "hub_small", "chol_smem", "chol_threads", "sb_elim", "n_sbe", "n_leaf", "hub0", "n_hub",
               "n_lc", "n_c", "ldw", "rec_stride", "gather_nosync", "row_tiles", "n_g12", "n_tile", "schur0", "schur1")
# DBG_LIN_JOBS: the kernel variants in launch_proj_lin's index order, the five counts kept for each, then two scalars
LIN_VARIANTS = ("proj_lin<2,2>", "proj_lin<4,2>", "proj_lin<2,4>", "proj_lin<4,4>",
                "pp<true,false>", "pp<false,false>", "pp<true,true>", "pp<false,true>")
LIN_JOBS_FIELDS = ("groups", "jobs", "tiles", "obs", "max_tiles_per_job")


class Config(C.Structure):
    _fields_ = [
        ("version", C.c_int32), ("device", C.c_int32), ("max_windows", C.c_int32),
        ("max_num_iterations", C.c_int32), ("consensus_max_steps", C.c_int32),
        ("use_cuda_graph", C.c_int32),
        ("focal_length", C.c_double), ("depth_sqrt_inf", C.c_double), ("gravity_norm", C.c_double),
        ("huber_delta", C.c_double),
        ("rho_frame_T", C.c_double), ("rho_frame_theta", C.c_double), ("rho_landmark", C.c_double),
        ("relaxation_alpha", C.c_double),
        ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
        ("min_relative_decrease", C.c_double), ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double), ("max_solver_time_in_seconds", C.c_double),
    ]


def default_config(**kw):
    """Defaults mirror config/tum/tum_single.yaml + d2vins/src/d2vins_params.{hpp,cpp}."""
    c = Config()
    c.version = D2BA_VERSION
    c.device = 0
    c.max_windows = 1
    c.max_num_iterations = 8          # tum_single.yaml:49
    c.consensus_max_steps = 0
    c.use_cuda_graph = 1
    c.focal_length = 460.0            # d2vins_params.hpp:26
    c.depth_sqrt_inf = 20.0
    c.gravity_norm = 9.805            # tum_single.yaml g_norm
    c.huber_delta = 1.0               # d2estimator.cpp:764
    c.rho_frame_T = 100.0             # tum_multi.yaml:53-54
    c.rho_frame_theta = 100.0
    c.rho_landmark = 1.0
    c.relaxation_alpha = 0.0
    for k, v in kw.items():
        setattr(c, k, v)
    return c


class Report(C.Structure):
    _fields_ = [
        ("total_iterations", C.c_int32), ("successful_steps", C.c_int32), ("termination", C.c_int32),
        ("succ", C.c_int32), ("total_time", C.c_double), ("initial_cost", C.c_double),
        ("final_cost", C.c_double), ("state_changes", C.c_double),
        ("final_gradient_max_norm", C.c_double), ("final_radius", C.c_double),
    ]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


proj_obs_dtype = np.dtype([
    ("type", "<i4"), ("cam_a", "<i4"), ("cam_b", "<i4"), ("reserved", "<i4"),
    ("frame_a", "<i8"), ("frame_b", "<i8"), ("landmark_id", "<i8"),
    ("pts_i", "<f8", 3), ("pts_j", "<f8", 3), ("vel_i", "<f8", 3), ("vel_j", "<f8", 3),
    ("td_i", "<f8"), ("td_j", "<f8"), ("depth", "<f8"),
], align=True)
assert proj_obs_dtype.itemsize == 160

track_obs_dtype = np.dtype([
    ("frame_id", "<i8"), ("camera_id", "<i4"), ("depth_mea", "<i4"),
    ("pt3d_norm", "<f8", 3), ("velocity", "<f8", 3), ("cur_td", "<f8"), ("depth", "<f8"),
], align=True)
assert track_obs_dtype.itemsize == 80

imu_dtype = np.dtype([
    ("frame_a", "<i8"), ("frame_b", "<i8"), ("sum_dt", "<f8"),
    ("delta_p", "<f8", 3), ("delta_q", "<f8", 4), ("delta_v", "<f8", 3),
    ("linearized_ba", "<f8", 3), ("linearized_bg", "<f8", 3),
    ("jacobian", "<f8", 225), ("covariance", "<f8", 225),
], align=True)
assert imu_dtype.itemsize == 8 * (3 + 16 + 450)

blockref_dtype = np.dtype([("kind", "<i4"), ("pad", "<i4"), ("id", "<i8")], align=True)
assert blockref_dtype.itemsize == 16


def blockrefs(pairs):
    a = np.zeros(len(pairs), dtype=blockref_dtype)
    for i, (k, i_d) in enumerate(pairs):
        a[i]["kind"] = k
        a[i]["id"] = i_d
    return a


def ptr(a, ctype=None):
    """Pointer to a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p) if ctype is None else a.ctypes.data_as(C.POINTER(ctype))
