/*
 * d2ba.h -- C ABI of libd2ba.so: the Hopper-native (sm_90a) sliding-window visual-inertial
 * bundle-adjustment solver that replaces the Ceres-backed hot path of D2SLAM's d2vins.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Each entry point names the reference
 * interface it replaces (paths relative to the D2SLAM tree):
 *
 *   d2ba_create / d2ba_destroy   <- CeresSolver / ConsensusSolver construction in
 *                                   D2Estimator::init                  (d2vins/src/estimator/d2estimator.cpp:49-54)
 *                                   + ceres options                    (d2vins/src/d2vins_params.cpp:140-160)
 *   d2ba_reset                   <- SolverWrapper::reset / ConsensusSolver::reset
 *                                                                      (d2common/src/solver/SolverWrapper.cpp:20-24,
 *                                                                       d2common/src/solver/ConsensusSolver.cpp:15-24)
 *   d2ba_set_blocks              <- parameter blocks handed to ceres through
 *                                   ResidualInfo::paramsPointerList    (d2common/include/d2common/solver/BaseParamResInfo.hpp:68-74)
 *                                   + constness/manifold decisions of D2Estimator::setStateProperties
 *                                                                      (d2vins/src/estimator/d2estimator.cpp:358-423)
 *   d2ba_add_proj                <- SolverWrapper::addResidual(Landmark*ResInfo / DepthResInfo)
 *                                                                      (d2vins/src/estimator/ParamResidualInfo.hpp:18-180,
 *                                                                       d2vins/src/estimator/d2estimator.cpp:796-874)
 *   d2ba_add_landmark_tracks     <- D2Estimator::setupLandmarkFactors  (d2vins/src/estimator/d2estimator.cpp:758-877)
 *   d2ba_add_imu                 <- SolverWrapper::addResidual(ImuResInfo) + IMUFactor ctor
 *                                                                      (d2vins/src/estimator/d2estimator.cpp:687-736,
 *                                                                       d2vins/src/factors/imu_factor.h:27-32)
 *   d2ba_set_prior               <- SolverWrapper::addResidual(PriorResInfo)
 *                                                                      (d2vins/src/estimator/d2estimator.cpp:888-897,
 *                                                                       d2vins/src/factors/prior_factor.cpp:45-90)
 *   d2ba_set_prior_info          <- PriorFactor ctor / toJacRes        (d2vins/src/factors/prior_factor.cpp:132-177)
 *   d2ba_set_consensus           <- ConsensusSolver::addParam + ConsensusSolverConfig
 *                                                                      (d2common/src/solver/ConsensusSolver.cpp:26-37,
 *                                                                       d2common/include/d2common/solver/ConsensusSolver.hpp:9-45)
 *   d2ba_comm_*                  <- D2VINSNet / LCM DISTRIB_VINS_DATA  (d2vins/src/network/d2vins_net.cpp:8-73,
 *                                                                       d2vins/src/estimator/solver/VINSConsenusSolver.cpp:11-120)
 *   d2ba_finalize                <- ceres::Problem::AddResidualBlock loop
 *                                                                      (d2common/src/solver/SolverWrapper.cpp:27-33)
 *   d2ba_solve                   <- CeresSolver::solve / ConsensusSolver::solve
 *                                                                      (d2common/src/solver/SolverWrapper.cpp:26-49,
 *                                                                       d2common/src/solver/ConsensusSolver.cpp:39-75)
 *   d2ba_get_blocks              <- in-place write-back through the raw double* blocks, read by
 *                                   D2EstimatorState::syncFromState    (d2vins/src/estimator/d2vinsstate.cpp:557-592)
 *   d2ba_report                  <- SolverReport                       (d2common/include/d2common/solver/SolverWrapper.hpp:14-37)
 *   d2ba_marginalize             <- Marginalizer::marginalize          (d2vins/src/estimator/marginalization/marginalization.cpp:173-254)
 *
 * Conventions
 *   - All floating point is IEEE binary64 (reference: state_type = double,
 *     d2common/include/d2common/d2basetypes.h:21).
 *   - pose / extrinsic block = [x y z qx qy qz qw] (7, tangent 6); speed-bias = [v ba bg] (9);
 *     inverse depth 1; td 1  (d2common/src/d2vinsframe.cpp:108-122, d2basetypes.h:7-14).
 *   - One handle owns a *batch* of independent "windows" (one window = the problem one
 *     D2Estimator hands to its solver).  window 0 of a max_windows=1 handle is the
 *     single-estimator drop-in.  Several windows on one handle are solved in the same
 *     kernel launches (throughput mode, or several agents of a swarm on one GPU).
 *   - The library copies every input during the call; the caller keeps ownership.
 *   - Every function returns 0 on success, non-zero on error (d2ba_last_error gives text).
 *     No exceptions cross this boundary.  There is no CPU fallback: without a CUDA device
 *     d2ba_create fails.
 *   - Threads: d2ba_set_blocks / d2ba_add_proj / d2ba_add_landmark_tracks / d2ba_add_imu / d2ba_set_prior* /
 *     d2ba_set_consensus may be called concurrently for DIFFERENT windows of one handle (one feeding thread per
 *     window at a time); everything else -- create, reset, finalize, solve*, get_blocks, marginalize, comm_*,
 *     debug_* -- must be called from one thread at a time with no feeding call in flight (the reference calls
 *     solve() under frame_mutex from one thread, d2estimator.cpp:324,529).  Different handles are independent.
 */
#ifndef D2BA_H_
#define D2BA_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define D2BA_VERSION 1

/* ---- parameter block kinds (reference ParamsType, BaseParamResInfo.hpp:7-17) ---- */
enum d2ba_block_kind {
  D2BA_POSE = 0,       /* frame pose, id = frame_id (int64)                   */
  D2BA_EXTRINSIC = 1,  /* camera extrinsic, id = camera_id                    */
  D2BA_SPEED_BIAS = 2, /* id = frame_id                                       */
  D2BA_TD = 3,         /* one per window, id ignored                          */
  D2BA_LANDMARK = 4    /* inverse depth in the anchor camera, id = landmark_id*/
};

/* ---- reprojection residual types (reference ResidualType, BaseParamResInfo.hpp:42-54) ---- */
enum d2ba_proj_type {
  D2BA_PROJ_2F1C = 0,      /* ProjectionTwoFrameOneCamFactor      <2;7,7,7,1,1>   */
  D2BA_PROJ_2F2C = 1,      /* ProjectionTwoFrameTwoCamFactor      <2;7,7,7,7,1,1> */
  D2BA_PROJ_1F2C = 2,      /* ProjectionOneFrameTwoCamFactor      <2;7,7,1,1>     */
  D2BA_PROJ_2F1C_DEPTH = 3,/* ProjectionTwoFrameOneCamDepthFactor <3;7,7,7,1,1>   */
  D2BA_PROJ_DEPTH_PRIOR = 4/* OneFrameDepth                       <1;1>           */
};

enum d2ba_termination {
  D2BA_TERM_NO_CONVERGENCE = 0, /* iteration budget exhausted            */
  D2BA_TERM_FUNCTION_TOL = 1,
  D2BA_TERM_GRADIENT_TOL = 2,
  D2BA_TERM_PARAMETER_TOL = 3,
  D2BA_TERM_FAILURE = 4         /* too many invalid steps / NaN          */
};

typedef struct d2ba_handle d2ba_handle;

typedef struct d2ba_config {
  int32_t version;             /* must be D2BA_VERSION                                   */
  int32_t device;              /* CUDA device ordinal                                    */
  int32_t max_windows;         /* batch capacity of the handle                           */
  int32_t max_num_iterations;  /* ceres max_num_iterations (d2vins_params.cpp:144)       */
  int32_t consensus_max_steps; /* 0 = plain solve (CeresSolver); >0 = ADMM sub-steps,
                                  each with max_num_iterations/steps iterations
                                  (d2vins_params.cpp:156-158)                            */
  int32_t use_cuda_graph;      /* capture the iteration sequence in a CUDA graph          */
  double focal_length;         /* projection sqrt_info = focal/1.5 (d2vins_params.cpp:172)*/
  double depth_sqrt_inf;       /* d2vins_params.cpp:178-180                               */
  double gravity_norm;         /* IMUData::Gravity = (0,0,g)                              */
  double huber_delta;          /* HuberLoss(1.0) d2estimator.cpp:764; <=0 disables        */
  /* ADMM (ConsensusSolverConfig, ConsensusSolver.hpp:9-22) */
  double rho_frame_T;
  double rho_frame_theta;
  double rho_landmark;
  double relaxation_alpha;
  /* trust-region constants (Ceres 2.1 defaults, SURVEY.md appendix B); 0 = default */
  double initial_trust_region_radius; /* 1e4  */
  double max_trust_region_radius;     /* 1e16 */
  double min_relative_decrease;       /* 1e-3 */
  double function_tolerance;          /* 1e-6 */
  double gradient_tolerance;          /* 1e-10 */
  double parameter_tolerance;         /* 1e-8 */
  /* ceres max_solver_time_in_seconds (d2vins_params.cpp:143; divided by consensus_max_steps per ADMM sub-step, :156-160):
   * no further trust-region iteration is started once the budget is used up (termination = NO_CONVERGENCE like ceres).
   * 0 = no budget.  d2ba_solve_fixed ignores it. */
  double max_solver_time_in_seconds;
} d2ba_config;

/* One reprojection residual block in reference terms: ids, not indices.
 * Fields unused by a type are ignored (cam_b for 2F1C, frame_b for 1F2C ...). */
typedef struct d2ba_proj_obs {
  int32_t type;        /* d2ba_proj_type                                            */
  int32_t cam_a;       /* camera_id of the anchor observation (extrinsic block a)   */
  int32_t cam_b;       /* camera_id of the second observation (2F2C, 1F2C)          */
  int32_t reserved;
  int64_t frame_a;     /* anchor frame (pose_i)                                     */
  int64_t frame_b;     /* observing frame (pose_j)                                  */
  int64_t landmark_id;
  double pts_i[3];     /* anchor bearing (LandmarkPerFrame::measurement, d2landmarks.h:166-168) */
  double pts_j[3];
  double vel_i[3];
  double vel_j[3];
  double td_i;         /* cur_td stamped at observation time                        */
  double td_j;
  double depth;        /* measured depth of observation j (DEPTH types), else 0     */
} d2ba_proj_obs;

/* One observation of a landmark track (reference LandmarkPerFrame, d2landmarks.h:28-120). */
typedef struct d2ba_track_obs {
  int64_t frame_id;
  int32_t camera_id;
  int32_t depth_mea;   /* 1 if depth is a valid measurement                        */
  double pt3d_norm[3]; /* unit-sphere bearing                                       */
  double velocity[3];
  double cur_td;
  double depth;
} d2ba_track_obs;

/* IMU pre-integration between consecutive frames (reference IntegrationBase,
 * d2common/include/d2common/integration_base.h:229-248). Matrices row-major 15x15,
 * state order P0 R3 V6 BA9 BG12. */
typedef struct d2ba_imu {
  int64_t frame_a;
  int64_t frame_b;
  double sum_dt;
  double delta_p[3];
  double delta_q[4];       /* x y z w */
  double delta_v[3];
  double linearized_ba[3];
  double linearized_bg[3];
  double jacobian[225];
  double covariance[225];
} d2ba_imu;

typedef struct d2ba_blockref {
  int32_t kind;  /* d2ba_block_kind */
  int32_t pad;
  int64_t id;
} d2ba_blockref;

typedef struct d2ba_report {     /* SolverReport, SolverWrapper.hpp:14-37 */
  int32_t total_iterations;      /* successful + unsuccessful steps (SolverWrapper.cpp:41-42) */
  int32_t successful_steps;
  int32_t termination;           /* d2ba_termination */
  int32_t succ;                  /* 1 unless failure */
  double total_time;             /* seconds, device time of the solve */
  double initial_cost;
  double final_cost;
  double state_changes;          /* |x_final - x_initial| over the free pose positions of the window (SolverReport.state_changes) */
  double final_gradient_max_norm;
  double final_radius;
} d2ba_report;

/* ---------------------------------------------------------------- lifecycle */
int d2ba_default_config(d2ba_config *cfg);
int d2ba_create(const d2ba_config *cfg, d2ba_handle **out);
int d2ba_destroy(d2ba_handle *h);
int d2ba_reset(d2ba_handle *h);
const char *d2ba_last_error(const d2ba_handle *h);

/* ---------------------------------------------------------------- problem input */
/* values: n * {7,7,9,1,1} doubles by kind.  is_const may be NULL (all free).  Calling it again
 * for an id that exists overwrites value/constness (used between solves). */
int d2ba_set_blocks(d2ba_handle *h, int32_t window, int32_t kind, int32_t n,
                    const int64_t *ids, const double *values, const uint8_t *is_const);
int d2ba_add_proj(d2ba_handle *h, int32_t window, int32_t n, const d2ba_proj_obs *obs);
/* Landmark tracks -> residual blocks with the reference's anchor / factor-type dispatch.
 * track_ptr has n_landmarks+1 entries indexing into obs.  fuse_dep/min/max depth as
 * D2VINSConfig (d2vins_params.hpp).  is_remote_frame callback-free form: frames listed in
 * ignore_frames (may be NULL) are skipped as d2estimator.cpp:776-794 does. */
int d2ba_add_landmark_tracks(d2ba_handle *h, int32_t window, int32_t n_landmarks,
                             const int64_t *landmark_ids, const int32_t *track_ptr,
                             const d2ba_track_obs *obs, int32_t fuse_dep,
                             double min_depth_to_fuse, double max_depth_to_fuse,
                             int32_t n_ignore_frames, const int64_t *ignore_frames);
int d2ba_add_imu(d2ba_handle *h, int32_t window, int32_t n, const d2ba_imu *imu);
/* Prior r = e0 + J*dx over the listed kept blocks.  J is m x m row-major, m = sum of
 * tangent sizes in refs order; x0 = linearisation points, concatenated nominal sizes. */
int d2ba_set_prior(d2ba_handle *h, int32_t window, int32_t m, const double *J,
                   const double *e0, int32_t nblk, const d2ba_blockref *refs,
                   const double *x0);
/* Same, from information form (A,b): performs the reference's toJacRes on the device. */
int d2ba_set_prior_info(d2ba_handle *h, int32_t window, int32_t m, const double *A,
                        const double *b, int32_t nblk, const d2ba_blockref *refs,
                        const double *x0);
/* Consensus slots: each listed POSE/EXTRINSIC block of this window takes part in the
 * ADMM averaging under global slot index slot[i] (shared by every window / rank that
 * holds the same frame_id / camera_id).  n_slots_global = size of the slot table. */
int d2ba_set_consensus(d2ba_handle *h, int32_t window, int32_t n, const d2ba_blockref *refs,
                       const int32_t *slot, int32_t n_slots_global);

/* ---------------------------------------------------------------- multi-GPU exchange */
/* 128-byte NCCL unique id made on rank 0 and distributed by the caller. */
int d2ba_comm_unique_id(uint8_t out[128]);
int d2ba_comm_init(d2ba_handle *h, const uint8_t unique_id[128], int32_t rank, int32_t nranks);
/* Pointer + element count of the device consensus buffer (f64, [n_slots][14] = sum p (3), sum vech(q q^T) (10), count):
 * a read-only view of what the last ADMM sub-step exchanged (tests, tracing).  The exchange itself always runs inside
 * d2ba_solve -- pack -> ncclAllReduce when a communicator is attached (d2ba_comm_init), local sum otherwise -> apply;
 * there is no step-wise entry point for an external transport.  A multi-process swarm WITHOUT d2ba_comm_init therefore
 * averages only the agents held by this handle. */
int d2ba_consensus_buffer(d2ba_handle *h, void **dev_ptr, int64_t *n_doubles);

/* ---------------------------------------------------------------- solve + output */
int d2ba_finalize(d2ba_handle *h);
int d2ba_solve(d2ba_handle *h, d2ba_report *reports /* [n windows in use], may be NULL */);
/* Run exactly `iters` trust-region iterations on every window without convergence exits
 * (benchmark / parity mode). */
int d2ba_solve_fixed(d2ba_handle *h, int32_t iters, d2ba_report *reports);
int d2ba_get_blocks(d2ba_handle *h, int32_t window, int32_t kind, int32_t n,
                    const int64_t *ids, double *values_out);
int d2ba_num_windows(const d2ba_handle *h);

/* ---------------------------------------------------------------- marginalization (next row, 8f-1) */
/* Marginalize the listed frames out of window `window` using the residuals currently added to it
 * (Marginalizer::marginalize with remove_base_when_margin_remote = 2, margin_enable_fej = 0, exact-inverse Schur
 * complement: config/tum/tum_single.yaml:87-94).  Returns the new prior in information form: A_out is
 * m_out x m_out row-major, b_out has m_out entries, refs_out lists the kept blocks (POSE, SPEED_BIAS, EXTRINSIC, TD
 * order, tangent sizes 6/9/6/1) and x0_out their linearisation points (concatenated nominal sizes 7/9/7/1).
 * Hand it back with d2ba_set_prior_info after the window has been rebuilt without the removed frames. */
int d2ba_marginalize(d2ba_handle *h, int32_t window, int32_t n_remove,
                     const int64_t *remove_frame_ids, int32_t *m_out, int32_t max_m,
                     double *A_out, double *b_out, int32_t *nblk_out, int32_t max_blk,
                     d2ba_blockref *refs_out, double *x0_out);

/* ---------------------------------------------------------------- introspection (parity tests) */
enum d2ba_debug_item {
  D2BA_DBG_N_CAM = 0,        /* reduced-camera dimension n_c (int64 scalar in out[0])        */
  D2BA_DBG_HCC = 1,          /* n_c x n_c row-major                                            */
  D2BA_DBG_GC = 2,           /* n_c                                                            */
  D2BA_DBG_HLL = 3,          /* L                                                              */
  D2BA_DBG_GL = 4,           /* L                                                              */
  D2BA_DBG_W = 5,            /* L x n_lc row-major (landmark-camera coupling)                  */
  D2BA_DBG_COST = 6,         /* scalar                                                         */
  D2BA_DBG_S = 7,            /* reduced system n_c x n_c                                       */
  D2BA_DBG_N_LC = 8,         /* landmark-coupled dimension (int64 scalar)                      */
  D2BA_DBG_OBS_INDEX = 9,    /* int32[6] per sorted obs: type, blk_i, blk_j, blk_ea, blk_eb, lm*/
  D2BA_DBG_COL_OF_BLOCK = 10,/* int32 column offset of every block, kind-major                 */
  D2BA_DBG_PROJ_RESJAC = 11, /* per obs (input order): r[3], J (3 x 27) row-major tangent      */
  D2BA_DBG_STEP = 12,        /* last trust-region step, n_c + L                                */
  D2BA_DBG_GN_STEP = 13,
  D2BA_DBG_IMU_RESJAC = 14,  /* per IMU factor (input order): r[15], J (15 x 30) row-major tangent columns
                                [pose_i 6 | speed-bias_i 9 | pose_j 6 | speed-bias_j 9], both times sqrt_info        */
  D2BA_DBG_CONS_RESJAC = 15  /* per six-dof block (poses then extrinsics, input order) 62 doubles: x[7], z[7], tilde[6],
                                r[6], J (6 x 6) row-major tangent of ConsenusPoseFactor at the current state; zeros for
                                blocks outside the consensus set                                                       */
};
/* Linearise at the current state (no step) so that the debug items are defined. */
int d2ba_debug_linearize(d2ba_handle *h);
int d2ba_debug_get(d2ba_handle *h, int32_t window, int32_t item, void *out, int64_t out_bytes,
                   int64_t *needed_bytes);
/* Device time (ms, CUDA events on the solver stream) of each kernel of the iteration sequence, summed over `iters`
 * iterations: [0] lm_gather (+ sb_elim), [1] reduced system (Schur tiles + leaf elimination), [2] dense Cholesky (+ sb / leaf back
 * substitution), [3] step, [4] misc_lin, [5] proj_lin, [6] control, [7] = iters, and the shares [8] sb_elim (of [0]),
 * [9] sb_back (of [2]), [10] leaf_elim (of [1]), [11] leaf_back (of [2]). */
int d2ba_debug_kernel_times(d2ba_handle *h, int32_t iters, double *ms_out /* [12] */);
/* Host wall-clock (ms) of the phases of the last d2ba_finalize: [plan (pair-major order, groups, jobs), prefix sums +
 * staging resize, staging fill, upload enqueue, error check, read-back buffers, device ms of the uploads, device ms of tile build + prep kernels], followed by
 * the thread-summed ms spent inside d2ba_add_proj since the last d2ba_reset: [id lookup, stamp scan, staging copy,
 * CUDA calls], then the host wall-clock ms of the last solve: [enqueue, wait for the device, write-back] and, in [15], the
 * host-to-device BYTES of the last reset -> add -> finalize cycle (observation records + staging arena). */
int d2ba_debug_host_times(d2ba_handle *h, double *ms_out /* [16] */);

#ifdef __cplusplus
}
#endif
#endif /* D2BA_H_ */
