/*
 * d2pgo.h -- C ABI of the pose-graph part of libd2ba.so: distributed Gauss-Newton / Levenberg-Marquardt over SE(3) poses
 * connected by relative-pose edges (BASELINE.json configs[4], SURVEY.md section 8f rank 3: "next" row after the BA path).
 *
 * What it stands in for in the reference (paths relative to the D2SLAM tree):
 *   d2pgo_create / d2pgo_destroy  <- D2PGO construction + the solver it owns           (d2pgo/src/d2pgo.cpp:155-256, :266)
 *   d2pgo_set_poses               <- PGOState frame pose blocks, fixed first frame      (d2pgo/src/pgostate.hpp:25-54)
 *   d2pgo_add_edges               <- setupLoopFactors / setupEgoMotionFactors           (d2pgo/src/d2pgo.cpp:413-528):
 *                                    one RelPoseFactorAD<6;7,7> per edge (pgo_use_autodiff) (d2common/include/d2common/solver/RelPoseFactor.hpp:68-135)
 *   d2pgo_comm_init               <- the PGO_Sync_Data exchange over ROS topic / d2comm / LCM (d2comm/src/d2comm.cpp:25-46)
 *   d2pgo_solve                   <- D2PGO::solve_single / solve_multi -> ceres::Solve   (d2pgo/src/d2pgo.cpp:155-256)
 *   d2pgo_get_poses               <- the optimised poses written back into PGOState
 *   d2pgo_set_poses_4d            <- PGOState::addFrame, 4-DoF branch: to_vector_xyzyaw   (d2pgo/src/pgostate.hpp:31-33)
 *   d2pgo_add_edges_4d            <- setupLoopFactors / setupEgoMotionFactors, 4-DoF branches (d2pgo/src/d2pgo.cpp:422-423,
 *                                    496-500): one RelPoseFactor4D per edge (RelPoseFactor.hpp:196-238)
 *   d2pgo_get_poses_4d            <- syncFromState: the optimised [x y z yaw] blocks
 *
 * Scope note: the reference solves the multi-agent graph with ARock (asynchronous dual updates, ARock.cpp:140-328) around
 * per-agent ceres problems; BASELINE's config asks for a *distributed Gauss-Newton* on the 8 GPUs of one box.  Here every
 * rank holds the whole pose vector (10k poses = 560 KB) and a shard of the edges; one LM iteration = linearise the local
 * edges, block-Jacobi preconditioned conjugate gradients on (J^T J + lambda D) dx = -J^T r with the matrix never formed
 * (y = J^T (J x) per edge), the per-rank partial products summed with one ncclAllReduce per CG iteration over NVLink.
 * All floating point is binary64.  pose = [x y z qx qy qz qw], tangent = [dp, dtheta], retraction of
 * PoseLocalParameterization (pose_local_parameterization.cpp:13-38).
 *
 * 4-DoF (config.pose_dof = 4, d2pgo's default pgo_pose_dof = PGO_POSE_4D, d2pgo_config.h:37): pose = [x y z yaw] with roll
 * and pitch taken as known (gravity-aligned frames), tangent = the 4-vector itself, retraction of PosAngleManifold::Plus
 * (angle_manifold.h:39-68: x + dx, yaw passed through NormalizeAngle, so the yaws of the poses a step moved are in
 * [-pi, pi)).  A handle serves one of the two: the 6-DoF setters / getters on a 4-DoF handle (and the reverse) return
 * non-zero with a d2pgo_last_error message; d2pgo_solve, d2pgo_comm_init and d2pgo_debug_edges serve both.
 */
#ifndef D2PGO_H_
#define D2PGO_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct d2pgo_handle d2pgo_handle;

typedef struct d2pgo_config {
  int32_t device;
  int32_t max_iterations;      /* LM iterations (ceres max_num_iterations of the PGO solver)            */
  int32_t pcg_max_iterations;  /* conjugate-gradient iterations per LM iteration                         */
  int32_t pose_dof;            /* 0 or 6: 6-DoF poses (RelPoseFactorAD); 4: [x y z yaw] (RelPoseFactor4D); else create fails */
  double pcg_tolerance;        /* relative residual |r| / |b| at which CG stops                          */
  double lambda0;              /* initial LM damping (relative to the block diagonal), 0 = Gauss-Newton   */
  double function_tolerance;   /* stop when the relative cost decrease of an accepted step is below       */
} d2pgo_config;

typedef struct d2pgo_report {
  int32_t iterations;          /* LM iterations run (accepted + rejected)                                 */
  int32_t accepted;
  int32_t pcg_iterations;      /* total CG iterations                                                     */
  int32_t converged;
  double initial_cost, final_cost;   /* 1/2 sum |r|^2                                                     */
  double device_ms;
} d2pgo_report;

int d2pgo_default_config(d2pgo_config *cfg);
int d2pgo_create(const d2pgo_config *cfg, d2pgo_handle **out);
int d2pgo_destroy(d2pgo_handle *h);
const char *d2pgo_last_error(const d2pgo_handle *h);
/* all poses of the graph (every rank gets the same list); fixed[i] != 0 keeps pose i constant (may be NULL) */
int d2pgo_set_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses7, const uint8_t *fixed);
/* relative-pose edges T_a^-1 T_b = rel: rel7 = [t, q(xyzw)], sqrt_info = 6x6 row-major applied to [dp ; 2 vec(dq)]
 * (RelPoseFactor.hpp:95-104).  With a communicator attached, each rank passes ITS shard of the edges. */
int d2pgo_add_edges(d2pgo_handle *h, int32_t n, const int64_t *id_a, const int64_t *id_b, const double *rel7, const double *sqrt_info36);
int d2pgo_comm_init(d2pgo_handle *h, const uint8_t unique_id[128], int32_t rank, int32_t nranks);
int d2pgo_solve(d2pgo_handle *h, d2pgo_report *report);
int d2pgo_get_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, double *poses7_out);
/* 4-DoF handles (pose_dof = 4): poses4 = [x y z yaw] */
int d2pgo_set_poses_4d(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses4, const uint8_t *fixed);
/* rel4 = [x y z yaw] of b in a's yaw frame, sqrt_info16 = 4x4 row-major applied to
 * [p_meas - Rz(-yaw_a)(p_b - p_a) ; NormalizeAngle(yaw_meas - NormalizeAngle(yaw_b - yaw_a))] (RelPoseFactor.hpp:218-227,
 * utils.hpp:240-280).  With a communicator attached, each rank passes ITS shard of the edges. */
int d2pgo_add_edges_4d(d2pgo_handle *h, int32_t n, const int64_t *id_a, const int64_t *id_b, const double *rel4, const double *sqrt_info16);
int d2pgo_get_poses_4d(d2pgo_handle *h, int32_t n, const int64_t *ids, double *poses4_out);
/* parity hook: residual and the two tangent Jacobians of every local edge at the current poses, row-major:
 * 6-DoF out[n_edges][78] = r(6) | J_a (6x6) | J_b (6x6);  4-DoF out[n_edges][36] = r(4) | J_a (4x4) | J_b (4x4) */
int d2pgo_debug_edges(d2pgo_handle *h, double *out, int64_t out_doubles);

#ifdef __cplusplus
}
#endif
#endif
