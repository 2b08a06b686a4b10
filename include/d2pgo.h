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
 *   d2pgo_pcm                     <- SwarmLocalOutlierRejection::OutlierRejectionLoopEdges (enable_pcm), the loops it keeps
 *                                    being those setupLoopFactors receives (d2pgo/src/d2pgo.cpp:177-186, :276-282)
 *   d2pgo_add_gravity_priors      <- setupGravityPriorFactors (enable_gravity_prior): GravityPriorPerturbAD per frame
 *                                    (d2pgo/src/d2pgo.cpp:530-559, GravityPrior.hpp:8-46)
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

/* ---- gravity prior (enable_gravity_prior, 6-DoF handles)
 *   d2pgo_add_gravity_priors <- D2PGO::setupGravityPriorFactors (d2pgo/src/d2pgo.cpp:530-559, called by solve_single /
 *                               solve_multi at :216-218, :304-306): one GravityPriorPerturbAD per frame
 *                               (d2common/include/d2common/solver/GravityPrior.hpp:8-46)
 * Per prior: pose i, its frame's ego (VIO) pose q_ego and a 3x3 S (row-major; d2pgo passes gravity_sqrt_info I3, 10 in the
 * shipped configs).  u = R(q_i)^T e3 (the third row of R_i), u_ego = R(q_ego)^T e3, and
 *     r = S^T (u - u_ego)      (the reference's row R_i.row(2) - R_ego.row(2) with applyOnTheRight(S))
 * with the tangent Jacobian dr/d dtheta = S^T [u]x, dr/d dp = 0: it ties roll and pitch to the observed gravity direction and
 * leaves yaw free.  Evaluated at the exact pose; the reference's perturbation chart q0 (x) quatfromRotationVector(theta) agrees
 * at theta = 0 and wherever |theta| >= 1e-2 (inside, its unnormalised [1, theta/2] is off by O(|theta|^2)).  A pose may carry
 * one prior; a fixed pose's prior only adds to the cost.  d2pgo_set_poses removes every prior.  With a communicator attached,
 * each rank passes ITS shard of the priors (each prior on exactly one rank).  Costs in d2pgo_report include the priors.
 * Returns 5 on a 4-DoF handle (d2pgo skips the prior for 4-DoF, d2pgo.cpp:531-533); 2 on an unknown id, a second prior on a
 * pose, a non-finite value or a zero ego quaternion (nothing of the call is kept); 1 on a null argument or n < 0.
 * d2pgo_last_error says why.  n = 0 changes nothing. */
int d2pgo_add_gravity_priors(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *ego_poses7, const double *sqrt_info9);
/* parity hook: per local prior at the current poses, in the order added, out[n_priors][21] = r(3) | J (3x6 row-major in the
 * tangent [dp, dtheta]; the position columns are zero) */
int d2pgo_debug_gravity_priors(d2pgo_handle *h, double *out, int64_t out_doubles);

/* ---- loop-closure outlier rejection: pairwise-consistency maximisation (PCM)
 *   d2pgo_pcm  <- SwarmLocalOutlierRejection::OutlierRejectionLoopEdges with redundant = true, incremental_pcm = false,
 *                 is_4dof = (pose_dof == 4), fed every loop once in the order given
 *                 (d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:46-303; called by D2PGO::solve_single /
 *                 solve_multi before setupLoopFactors, d2pgo/src/d2pgo.cpp:177-186, :276-282, when enable_pcm is set)
 *   clique     <- FMC::maxCliqueHeu (d2pgo/third_party/fast_max-clique_finder/src/findCliqueHeu.cpp:124-243)
 * Loops are grouped by the unordered pair of drone ids (a drone with itself included).  Within a group every loop i is tested
 * against every earlier loop j: err = odom_a p2 odom_b^-1 rel_i^-1 with p2 = rel_j, odom_a = odom(a_i -> a_j), odom_b =
 * odom(b_i -> b_j) when the two loops name the drones in the same order, and p2 = rel_j^-1, odom_a = odom(a_i -> b_j), odom_b =
 * odom(b_i -> a_j) when swapped; smd = log(err)^T Sigma^-1 log(err), Sigma = cov_i + cov_j + cov(odom_a) + cov(odom_b), and the
 * two loops are consistent iff smd < (float)pcm_thres.  A loop is an inlier iff it is in its group's FMC clique.
 * odom(f -> g) = DeltaPose(ego_f, ego_g) (yaw only on a 4-DoF handle: (Rz(-yaw_f)(p_g - p_f), Rz(yaw_g - yaw_f))) with the
 * diagonal covariance (pos_covariance_per_meter len + yaw_covariance_per_meter len^2 / 2) I3, yaw_covariance_per_meter len I3
 * at the path length len along the drone's keyframes between f and g (a drone's keyframes in the order given).
 * cov_i = (S^T S)^-1 of the loop's 6x6 square-root information; log = [t ; rotation vector].
 * The handle's poses and edges are not touched: add the inliers with d2pgo_add_edges[_4d].  Deterministic (bitwise the same
 * mask on every call and every rank).  A group holds at most 32768 loops. */
typedef struct d2pgo_pcm_config {
  double pcm_thres;                  /* consistency threshold on smd; rounded to float like the reference's field (1.635) */
  double pos_covariance_per_meter;   /* ego-motion model (d2pgo_config.h defaults 4e-3, 4e-5)                          */
  double yaw_covariance_per_meter;
} d2pgo_pcm_config;

typedef struct d2pgo_pcm_report {
  int32_t groups;                    /* drone pairs with at least one loop                                              */
  int32_t inliers;
  int64_t pairs_tested;              /* sum over groups of L (L - 1) / 2                                                */
  int64_t consistent_pairs;
  int64_t clique_rounds;             /* greedy picks made by the clique kernel, seeds examined again included           */
  double device_ms, pair_ms, clique_ms;   /* whole call on the device; its consistency part; its clique part          */
} d2pgo_pcm_report;

int d2pgo_default_pcm_config(d2pgo_pcm_config *cfg);
/* frames: every keyframe a loop names, with its drone and ego (odometry) pose [x y z qx qy qz qw]; loops: keyframe ids,
 * rel7 = T_a^-1 T_b, sqrt_info36 row-major.  inlier_out[n_loops] = 1 / 0.  Returns non-zero (d2pgo_last_error says why) on
 * an unknown or duplicate keyframe id, a non-finite or non-positive threshold, or a group of more than 32768 loops. */
int d2pgo_pcm(d2pgo_handle *h, const d2pgo_pcm_config *cfg, int32_t n_frames, const int64_t *frame_ids, const int32_t *frame_agent,
              const double *ego_poses7, int32_t n_loops, const int64_t *kf_a, const int64_t *kf_b, const double *rel7,
              const double *sqrt_info36, uint8_t *inlier_out, d2pgo_pcm_report *report);
/* parity hooks.  smd of every tested pair (i, j < i) of the last d2pgo_pcm call: groups in order of their first loop, rows i
 * ascending, j ascending (report.pairs_tested doubles).  The clique kernel alone on a caller-given symmetric adjacency without
 * self loops, adj[n][ceil(n / 32)] words, bit j of row i = word j / 32, bit j % 32: member_out[n], size_out = clique size. */
int d2pgo_debug_pcm_smd(d2pgo_handle *h, double *out, int64_t out_doubles);
int d2pgo_debug_pcm_clique(d2pgo_handle *h, int32_t n, const uint32_t *adj, uint8_t *member_out, int32_t *size_out);

#ifdef __cplusplus
}
#endif
#endif
