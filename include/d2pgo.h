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
 *   d2pgo_pcm_stream[_reset]      <- the same object kept across solves: only the loops new in each call are tested (below)
 *   d2pgo_add_gravity_priors      <- setupGravityPriorFactors (enable_gravity_prior): GravityPriorPerturbAD per frame
 *                                    (d2pgo/src/d2pgo.cpp:530-559, GravityPrior.hpp:8-46)
 *   d2pgo_arock_*                 <- ARockPGO, d2pgo's distributed pgo_mode 1 (ARock.cpp:24-314, ARockPGO.cpp:7-104; below)
 *   d2pgo_arock_rot_*             <- RotationInitARock, the rotation initialisation d2pgo runs before the ARock solve
 *                                    (rotation_initialization_arock.hpp:10-236; below)
 *
 * Scope note: the reference solves the multi-agent graph with ARock (dual updates around per-agent ceres problems,
 * ARock.cpp:140-328), which the d2pgo_arock_* entry points reproduce, one handle per agent.  BASELINE's config also asks for
 * a *distributed Gauss-Newton* on the 8 GPUs of one box, which d2pgo_comm_init provides: every
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

/* ---- PCM as a stream: the stateful object the reference node keeps between solves
 *   d2pgo_pcm_stream_reset  <- a new SwarmLocalOutlierRejection (redundant = true, is_4dof = (pose_dof == 4)) over empty
 *                              trajectories (d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:20-30)
 *   d2pgo_pcm_stream        <- one OutlierRejectionLoopEdges call with available_loops = the loops given
 *                              (swarm_outlier_rejection.cpp:46-120; D2PGO::solve_single / solve_multi pass every loop they
 *                              hold on each call, d2pgo/src/d2pgo.cpp:170-186), after the keyframes new since the last call
 *                              were pushed to their drones' trajectories
 *   incremental = 0         <- incremental_pcm = false: FMC::maxCliqueHeu on each group that got new loops (:287-301)
 *   incremental = 1         <- incremental_pcm = true (the d2pgo_config.h default): FMC::maxCliqueHeuIncremental's search
 *                              (d2pgo/third_party/fast_max-clique_finder/src/findCliqueHeuInc.cpp:32-96, :269-281)
 * A loop is tested only the first time its id appears, against every earlier loop of its group (edge1 = the new loop), with
 * d2pgo_pcm's consistency test; the consistency graph stays on the device between calls.  Only groups that got new loops run
 * the clique again; the others keep their inlier sets.  Mode 0 gives, after any split of an input into calls, the mask and
 * the smd d2pgo_pcm gives on the concatenated input.  Mode 1 seeds only the new vertices, starts from m = the group's clique
 * size, and replaces the group's set when a seed's clique beats m.
 * Declared deviation (mode 1): the reference copies FMC's candidate buffer v_i_S into the result (findCliqueHeuInc.cpp:92-94),
 * which is not the clique; here the set is the clique the search found, seed and picks, and its size is FMC's return value.
 * inlier_out[n_loops] = the call's loops that are in their group's set (:96-111; every group the stream holds has a set).
 * The stream is independent of d2pgo_pcm's buffers: calls to the two may interleave.  Deterministic, no atomics.
 * Refusals keep nothing of the call (the stream is as before it) and set d2pgo_last_error: 5 before any reset; 3 on a loop
 * naming an unknown keyframe, a loop id twice in one call, or a keyframe id given again with another drone; 2 on a non-finite
 * ego pose, relative pose or sqrt_info of a new frame or loop; 4 on a group growing past 32768 loops; 1 on a null argument. */
typedef struct d2pgo_pcm_stream_report {
  int32_t new_loops, total_loops;    /* loops first seen in this call; loops in the stream                              */
  int32_t groups, groups_touched;    /* drone pairs in the stream; those that got new loops                             */
  int32_t inliers;                   /* over the loops passed to this call                                              */
  int64_t pairs_tested, consistent_pairs, clique_rounds;   /* this call only                                           */
  double device_ms, pair_ms, clique_ms;
} d2pgo_pcm_stream_report;

/* forgets every frame, loop and clique.  cfg as for d2pgo_pcm; incremental 0 or 1 (above). */
int d2pgo_pcm_stream_reset(d2pgo_handle *h, const d2pgo_pcm_config *cfg, int32_t incremental);
/* frames: keyframes new since the last call, appended to their drone's trajectory in the order given (a keyframe id already in
 * the stream is ignored when it names the same drone).  loops: the call's available_loops keyed by loop_ids; an id seen
 * before is not tested again and its other fields are ignored. */
int d2pgo_pcm_stream(d2pgo_handle *h, int32_t n_frames, const int64_t *frame_ids, const int32_t *frame_agent, const double *ego_poses7,
                     int32_t n_loops, const int64_t *loop_ids, const int64_t *kf_a, const int64_t *kf_b, const double *rel7,
                     const double *sqrt_info36, uint8_t *inlier_out, d2pgo_pcm_stream_report *report);
/* parity hooks.  The smd of the pairs tested by the last stream call (report.pairs_tested doubles): groups in order of their
 * first loop, new rows i ascending, j < i ascending.  The incremental clique kernel alone on a caller-given adjacency (as
 * d2pgo_debug_pcm_clique) whose last n_new vertices are new, under the bound prev_size: member_out = the clique found when a
 * seed beats prev_size, else all 0; size_out = FMC::maxCliqueHeuIncremental's return value (n_new = n, prev_size = 0 is
 * maxCliqueHeu). */
int d2pgo_debug_pcm_stream_smd(d2pgo_handle *h, double *out, int64_t out_doubles);
int d2pgo_debug_pcm_clique_inc(d2pgo_handle *h, int32_t n, const uint32_t *adj, int32_t n_new, int32_t prev_size, uint8_t *member_out,
                               int32_t *size_out);

/* ---- ARock distributed mode (d2pgo's pgo_mode 1: PGO_MODE_DISTRIBUTED_AROCK)
 *   d2pgo_arock_enable     <- ARockPGO construction with ARockSolverConfig (d2common/include/d2common/solver/ARock.hpp:6-19)
 *   d2pgo_arock_receive    <- ARockPGO::inputDPGOData; processed at the next step as receiveAll / processPGOData
 *                             (d2pgo/src/ARockPGO.cpp:7-70)
 *   d2pgo_arock_step       <- one pass of ARockBase::solve_arock with max_steps = 1, as d2pgo_node runs it
 *                             (d2common/src/solver/ARock.cpp:140-190)
 *   d2pgo_arock_neighbours,
 *   d2pgo_arock_duals      <- ARockPGO::broadcastData: one message per neighbour, target = that neighbour (ARockPGO.cpp:72-104)
 * One handle is one agent (self_id).  Its poses and edges are that agent's sub-graph (D2PGO::solve_multi: its own ego-motion
 * edges and every loop whose two frames it knows); every pose carries its owner agent.  The dual table is keyed by
 * (neighbour agent, frame id) and holds a local dual y_l and a remote dual y_r, in dual coordinates:
 *   4-DoF handles: [x y z yaw] (POSE_4D);
 *   6-DoF handles: [p ; theta] with R = R(q_init) Exp(theta), theta = Log(q_init^-1 q) the principal log (POSE_PERTURB_6D,
 *                  d2pgo/src/pgostate.hpp:35-46; the node's perturb_mode).  q_init is the frame's attitude when it was added.
 *   6-DoF handles in the perturbation chart (d2pgo_set_chart): the state [p ; theta] itself, with the chart's proximal term
 *                  below.
 * One step:
 *   1. the received messages in arrival order: for a frame the local problem uses (an edge or a gravity prior touches it),
 *      if target == self_id or there is no dual (sender, frame) yet: create it with y_l = y_r = the value, or else set y_r;
 *   2. every frame the local problem uses and another agent d owns gets a dual (d, frame) if it has none, y_l = y_r = the
 *      frame's pose in dual coordinates (or 0 with dual_state_init_to_zero);
 *   3. the LM solve of d2pgo_solve over the edges, the gravity priors and one proximal term per dual, towards its y_r:
 *        4-DoF ConsenusPoseFactor4D (norm_yaw): r = diag(rho_T I3, rho_theta) [y_p - p ; N(N(y_yaw) - yaw)]  (weights rho,
 *              not sqrt(rho); d2common/include/d2common/solver/consenus_factor_4d.h)
 *        6-DoF NormalPrior: r = diag(sqrt(rho_T) I3, sqrt(rho_theta) I3) ([p ; theta] - y_r)   (ARock.cpp:284-291)
 *   4. updateDualStates (ARock.cpp:50-81) on every dual at the solved poses x (in dual coordinates):
 *        y_l -= eta_k ((y_l + y_r) / 2 - x), and on 4-DoF handles y_l's yaw normalised only when it lies outside [-pi, pi].
 * Only the fixed flags of d2pgo_set_poses hold the gauge: d2pgo fixes main_id's head frame and nothing else
 * (d2pgo/src/d2pgo.cpp:602-612).  The report is the local LM solve's (costs include the proximal terms).  d2pgo_set_poses
 * keeps the duals of the frames still present and every queued message; d2pgo_solve on an ARock handle solves its sub-graph
 * without proximal terms.  A handle in ARock mode refuses d2pgo_comm_init (5) and a handle with a communicator refuses
 * d2pgo_arock_enable (5).  Every refusal keeps nothing of the call and sets d2pgo_last_error. */
typedef struct d2pgo_arock_config {
  int32_t self_id;
  int32_t dual_state_init_to_zero;       /* ARockSolverConfig default 0                                              */
  double rho_frame_T, rho_frame_theta;   /* defaults 0.1 / 0.1; config/realsense_d435/d435_multi.yaml: 0.7 / 0.625   */
  double eta_k;                          /* default 0.9; d435_multi.yaml: 0.1                                        */
} d2pgo_arock_config;

int d2pgo_default_arock_config(d2pgo_arock_config *cfg);
/* owner agent of each pose id (ids must be poses of the handle; a later call adds to or replaces the table and the config).
 * 6-DoF: q_init4[n][4] (xyzw, normalised here), NULL = the attitude of the pose as d2pgo_set_poses gave it.  Returns 1 on a
 * null argument or n < 0, 2 on an unknown id, a non-finite or zero q_init or a bad config, 5 with a communicator attached. */
int d2pgo_arock_enable(d2pgo_handle *h, const d2pgo_arock_config *cfg, int32_t n, const int64_t *ids, const int32_t *owner,
                       const double *q_init4);
/* one message (sender, target, frames, duals[n][dim]), queued for the next step; dim must be 4 (4-DoF) or 6 (6-DoF).
 * Returns 2 on a wrong dim, a non-finite dual, a frame id twice, or sender == self_id; 5 if not in ARock mode. */
int d2pgo_arock_receive(d2pgo_handle *h, int32_t sender, int32_t target, int32_t n, const int64_t *frame_ids, int32_t dim,
                        const double *duals);
/* one ARock step; every pose needs an owner (and, 6-DoF, a q_init) */
int d2pgo_arock_step(d2pgo_handle *h, d2pgo_report *report);
/* the neighbours the dual table holds, ascending; *n_out = their number (2 if more than max_n) */
int d2pgo_arock_neighbours(d2pgo_handle *h, int32_t max_n, int32_t *n_out, int32_t *ids_out);
/* the broadcast payload for one neighbour: frame ids ascending, y_l [n][D] and (remote_out may be NULL) y_r [n][D];
 * *n_out = the count (2 if more than max_n) */
int d2pgo_arock_duals(d2pgo_handle *h, int32_t neighbour, int32_t max_n, int32_t *n_out, int64_t *frame_ids, double *local_out,
                      double *remote_out);
/* parity hook: per dual in table order ((neighbour, frame id) ascending), at the current poses and towards its y_r:
 * out[n_duals][D + D*D] = r (D) | J (D x D row-major, in the tangent: 4-DoF the 4-vector, 6-DoF [dp, dtheta] of the right
 * perturbation q (x) Exp(dtheta); the 6-DoF theta block is sqrt(rho_theta) J_r^-1(theta)) */
int d2pgo_debug_arock_terms(d2pgo_handle *h, double *out, int64_t out_doubles);

/* ---- chordal rotation initialisation (d2pgo's rotInitial, enable_rotation_initialization = true by default)
 *   d2pgo_rot_init  <- RotationInitialization<double>::solve on the non-distributed path (RotInit,
 *                      d2pgo/src/rot_init/rotation_initialization.cpp:21-28; rotation_initialization_base.hpp:440-456),
 *                      fed every edge of the handle (D2PGO::rotInitial's used_loops, d2pgo/src/d2pgo.cpp:336-361) and the
 *                      handle's fixed flags (the fixed frame, :346-349)
 * Unknowns: the three rows r_f^k of R_f of every free frame an edge names (updateFrameIdx, :57-69).  Per edge with rotation
 * weight s = |S[3:6, 3:6]|_F (the reference replaces each square-root block by its Frobenius norm times I3):
 *   a, b free, a != b:   s (R_ab^T r_a^k - r_b^k) = 0                     (setupRotInitProblembyLoop, :89-111)
 *   a fixed, b free:     s r_b^k = s (row k of R_a R_ab)^T                 (setPriorFactorsbyFixedParam, :72-87; ASSUMED: the
 *                        prior's rotation square root is that of the edge, so these are the edge rows with r_a held)
 *   a free, b fixed:     no rows -- the reference attaches that prior to frame b, the fixed frame, which has no unknowns (:84)
 *   both fixed, a == b:  no rows (:96-102)
 *   enable_gravity_prior: per free frame an edge names, g (r_f^2 - R_ego,f^T e3) = 0, e3 = (0, 0, 1) (:131-144)
 * The weights are scalar times I3, so the system splits into three 3N x 3N systems, one per k, sharing the edge structure;
 * the gravity rows enter k = 2 only.  Each is solved by the block-Jacobi PCG of d2pgo_solve (one Gauss-Newton step from zero,
 * D = 3 per frame) to pcg_tolerance; the reference factorises A^T A (SimplicialLLT, :146-176).  Each free frame then gets
 * R_f = U diag(1, 1, det(U V^T)) V^T of the SVD of its solved M_f = [r^0 r^1 r^2]^T (recoverRotationLLT :360-389,
 * Utility::recoverRotationSVD); its attitude becomes the quaternion of R_f (the sign may differ from the reference's) and its
 * position keeps every bit.  Fixed frames and frames no edge names keep their poses.  The edges, gravity priors and every
 * other table of the handle are untouched, so d2pgo_solve can follow directly.  Binary64, no atomics, bitwise reproducible.
 * Refusals keep nothing of the call and set d2pgo_last_error: 5 on a 4-DoF handle (a 4-DoF PGOState has no rotation states,
 * pgostate.hpp:31-47), with a communicator attached or in ARock mode (the reference runs RotationInitARock there); 2 when a
 * component of free frames (joined by the edges that give rows) holds no fixed frame -- A^T A is singular there and the
 * reference asserts (:173); a free frame named only by dropped edges is such a component --, when gravity rows are on and a
 * free frame lacks an ego pose, and on an unknown or duplicate ego id or a non-finite value; 1 on a null argument or n < 0. */
typedef struct d2pgo_rot_init_config {
  int32_t enable_gravity_prior;   /* RotInitConfig::enable_gravity_prior (d2pgo_config.h:11; d2pgo_test.cpp turns it on)   */
  int32_t pcg_max_iterations;     /* per row system k (default 20000)                                                       */
  double gravity_sqrt_info;       /* RotInitConfig default 10                                                               */
  double pcg_tolerance;           /* relative residual |A^T A x - A^T b| / |A^T b| at which CG stops (default 1e-12)        */
} d2pgo_rot_init_config;

typedef struct d2pgo_rot_init_report {
  int32_t frames;                 /* free frames solved                                                                     */
  int32_t edges_used, edges_dropped;   /* dropped: b fixed with a free, both fixed, self loops                              */
  int32_t pcg_iterations[3];      /* per row system k                                                                       */
  double residual[3];             /* relative residual reached per row system (CG recurrence)                               */
  double state_changes;           /* mean over free frames of |R_before - M_f|_F / |R_before|_F (SolverReport, :376-388)    */
  double device_ms;
} d2pgo_rot_init_report;

int d2pgo_default_rot_init_config(d2pgo_rot_init_config *cfg);
/* ego attitudes are read only with enable_gravity_prior (every free frame an edge touches needs one): ego_poses7[n_ego][7] of
 * the frames ego_ids, [x y z qx qy qz qw] (the attitude is normalised).  report may be NULL. */
int d2pgo_rot_init(d2pgo_handle *h, const d2pgo_rot_init_config *cfg, int32_t n_ego, const int64_t *ego_ids,
                   const double *ego_poses7, d2pgo_rot_init_report *report);

/* ---- distributed chordal rotation initialisation (d2pgo's rotInitial in pgo_mode 1: RotationInitARock<double>)
 *   d2pgo_arock_rot_init_step  <- one RotationInitARock::solve with max_steps = 1, one pass of ARockBase::solve_arock
 *                                 (d2pgo/src/rot_init/rotation_initialization_arock.hpp:195-205, d2common/src/solver/ARock.cpp:
 *                                 140-190), as D2PGO::rotInitial runs it (d2pgo/src/d2pgo.cpp:336-361)
 *   d2pgo_arock_rot_receive    <- RotationInitARock::inputDPGOData (:216-235); its duals are handled at the next step
 *   d2pgo_arock_rot_neighbours,
 *   d2pgo_arock_rot_duals      <- broadcastData (:113-140): one DPGO_ROT_MAT_DUAL message per neighbour of the table
 * On a 6-DoF handle in ARock mode (d2pgo_arock_enable: self_id, owners, eta_k).  The unknowns are the rows r_f^k of M_f of
 * every free frame an edge names, whoever owns it; only the handle's fixed flags fix frames (d2pgo fixes main_id's head frame,
 * d2pgo.cpp:346-349).  The rotation dual table is the handle's own, apart from the pose dual table of d2pgo_arock_step: keyed
 * (neighbour, frame id), ascending, y_l and y_r being 3x3 matrices stored row-major (9 doubles); d2pgo_set_poses keeps the
 * duals of the frames still present.  Every named frame has a rotation state R_state: R(attitude) when the frame first enters
 * a step, then the last unprojected M of that frame.  One step:
 *   1. receiveAll / processPGOData (:104-111, :142-182): the queued messages in arrival order; for a frame an edge names, if
 *      target == self_id or there is no dual (sender, frame) yet: the dual is created with zeros if missing, y_r = the value,
 *      and y_l = the value too if it was just created;
 *   2. the fixed-frame edge rows of d2pgo_rot_init (prepareSolverInIter :74-77, the :84 quirk included);
 *   3. scanAndCreateDualStates (:79-102): every edge end another agent owns gets the dual (owner, frame), zero, if it has none;
 *   4. setDualStateFactors (:32-61): per dual on a free frame, w (r_f^k - (row k of Y_r)^T) = 0, w = sqrt(3 rho_rot_mat)
 *      (ASSUMED: PosePrior's 3x3 argument rho I3 is information whose Cholesky factor is the square root, so
 *      |getSqrtInfoMatRot()|_F = sqrt(3 rho); and getRotMat() returns Y_r unprojected);
 *   5. solveLinearRot (rotation_initialization_base.hpp:178-213): the three row systems of d2pgo_rot_init over the edge rows,
 *      the fixed-frame rows and the dual priors, plus with enable_gravity_prior the gravity rows of every free frame, owned or
 *      remote (:195-201), by the block-Jacobi PCG to pcg_tolerance;
 *   6. recoverRotationLLT (:360-389) per free frame: state_changes += |R_state - M_f|_F / |R_state|_F, R_state = M_f; frames
 *      this agent owns take the attitude of R_f = U diag(1, 1, det(U V^T)) V^T (the zero matrix projects to I, as Eigen's
 *      JacobiSVD gives U = V = I there) and their ARock q_init becomes it; the report's state_changes is the mean;
 *   7. updateDualStates, vector branch (ARock.cpp:63-81), every dual: y_l -= eta_k ((y_l + y_r) / 2 - R_state of its frame)
 *      (for a fixed frame R_state is the rotation of its attitude when it entered).
 * Receipt (d2pgo_arock_rot_receive): every frame of the message that the handle holds and the sender owns takes the sender's
 * pose, position and attitude, and its q_init becomes that attitude; frames the handle does not hold are ignored.  So the first
 * d2pgo_arock_step after rotation initialisation starts from theta = 0 at the attitudes it left.  D2PGO::rotInitial declares
 * convergence once state_changes < rot_init_state_eps after more than 10 solves.  Binary64, no atomics, bitwise reproducible.
 * Refusals keep nothing of the call and set d2pgo_last_error: 5 on a 4-DoF handle or a handle not in ARock mode, and for a
 * step or a receipt once the pose dual table is non-empty (rotation initialisation precedes the perturbation solve); 2 on a component of free frames with
 * no fixed-frame edge row and no dual prior (gravity rows anchor k = 2 only; the reference asserts there), when gravity rows
 * are on and a free frame lacks an ego pose, on a dual dimension other than 9, a non-finite value, a zero quaternion, a frame
 * twice in one message or a message from self_id; 1 on a null argument or a negative count.  d2pgo_rot_init keeps refusing
 * ARock handles (5). */
typedef struct d2pgo_arock_rot_init_config {
  int32_t enable_gravity_prior;   /* RotInitConfig::enable_gravity_prior                                                   */
  int32_t pcg_max_iterations;     /* per row system k (default 20000)                                                      */
  double gravity_sqrt_info;       /* default 10                                                                            */
  double pcg_tolerance;           /* relative residual per row system (default 1e-12)                                      */
  double rho_rot_mat;             /* ARockSolverConfig::rho_rot_mat, default 0.1 (ARock.hpp:11); d2pgo_test_multi: 0.16      */
} d2pgo_arock_rot_init_config;

int d2pgo_default_arock_rot_init_config(d2pgo_arock_rot_init_config *cfg);
/* one step; ego_poses7[n_ego][7] of ego_ids as for d2pgo_rot_init (every free frame an edge names, owned or remote, needs one
 * with gravity rows on).  report may be NULL; its state_changes is 0 when there is no free frame. */
int d2pgo_arock_rot_init_step(d2pgo_handle *h, const d2pgo_arock_rot_init_config *cfg, int32_t n_ego, const int64_t *ego_ids,
                              const double *ego_poses7, d2pgo_rot_init_report *report);
/* one message: frames, duals[n][dim] (dim must be 9) and the sender's poses7[n][7] of those frames */
int d2pgo_arock_rot_receive(d2pgo_handle *h, int32_t sender, int32_t target, int32_t n, const int64_t *frame_ids, int32_t dim,
                            const double *duals, const double *poses7);
/* the neighbours of the rotation dual table, ascending; *n_out = their number (2 if more than max_n) */
int d2pgo_arock_rot_neighbours(d2pgo_handle *h, int32_t max_n, int32_t *n_out, int32_t *ids_out);
/* the broadcast payload for one neighbour: frame ids ascending, y_l [n][9], (may be NULL) y_r [n][9] and this handle's current
 * poses [n][7] of those frames; *n_out = the count (2 if more than max_n) */
int d2pgo_arock_rot_duals(d2pgo_handle *h, int32_t neighbour, int32_t max_n, int32_t *n_out, int64_t *frame_ids, double *local9,
                          double *remote9, double *poses7);
/* parity hook: per pose, state9_out[N][9] its R_state (0 before it entered a step) and flag_out[N] 0 = no edge names it,
 * 1 = free, 2 = fixed; the rotation dual table in table order: *n_duals_out entries (2 if more than max_duals) */
int d2pgo_debug_arock_rot_state(d2pgo_handle *h, double *state9_out, uint8_t *flag_out, int32_t max_duals, int32_t *n_duals_out,
                                int32_t *neighbour_out, int64_t *frame_out, double *local9_out, double *remote9_out);

/* ---- linear solver of the LM steps (the reference's ceres linear_solver_type)
 *   D2PGO_LINEAR_PCG             the default: (J^T J + lambda diag D) dx = -g by block-Jacobi PCG to pcg_tolerance, at most
 *                                pcg_max_iterations (a truncated step); the only kind with a communicator and for rot init.
 *                                d2pgo_debug_pcg_step takes one such step alone
 *   D2PGO_LINEAR_SPARSE_CHOLESKY <- SPARSE_NORMAL_CHOLESKY, which d2pgo uses for every pose graph (d2pgo/src/d2pgo_node.cpp:
 *                                191-195, and the ARock local solves, :202): the exact step from a supernodal multifrontal
 *                                Cholesky of H = J^T J + lambda diag(D) + 1e-12 I over the free poses, H being exactly the
 *                                operator PCG applies (self loops included).  Ordering by nested dissection, once per graph
 *                                structure on the host; factorisation and triangular solves on the device, binary64, no
 *                                atomics, bitwise reproducible.  A non-positive or non-finite pivot makes the step a rejected
 *                                one (lambda -> 4 lambda, or 1e-4 from 0).  pcg_iterations stays 0; pcg_* fields are unused.
 * The kind applies to d2pgo_solve and d2pgo_arock_step, 4-DoF and 6-DoF, with or without gravity priors; d2pgo_rot_init keeps
 * PCG.  It may change between solves.  Returns 2 on an unknown kind, 5 for the sparse Cholesky on a handle with a
 * communicator (and d2pgo_comm_init returns 5 on a sparse-Cholesky handle); a refusal keeps nothing.  A solve refuses (7,
 * before any device work, d2pgo_last_error says why) a structure with a front above 1024 scalar rows or whose fronts need
 * more than half the free device memory.  Switching back to PCG frees the factor's device memory and graphs. */
enum { D2PGO_LINEAR_PCG = 0, D2PGO_LINEAR_SPARSE_CHOLESKY = 1 };

typedef struct d2pgo_cholesky_info {
  int32_t free_poses;
  int32_t block_pairs;                    /* distinct pairs of free poses an edge joins (self loops excluded)           */
  int64_t nnz_L;                          /* D x D blocks of L, diagonal included (the exact symbolic count)             */
  int64_t nnz_L_stored;                   /* blocks stored after relaxed amalgamation (explicit zeros included)          */
  int32_t supernodes, levels;             /* of the amalgamated supernodal tree: one launch per level and phase          */
  int32_t supernodes_fundamental, levels_fundamental;   /* before amalgamation                                          */
  int32_t max_front_rows, max_front_cols; /* scalar                                                                      */
  int32_t factorizations, failed_factorizations;       /* during the last solve                                          */
  double factor_ms, solve_ms;             /* device ms of the factorisations (assembly included) and of the triangular
                                             solves, summed over the last solve                                          */
} d2pgo_cholesky_info;

int d2pgo_set_linear_solver(d2pgo_handle *h, int32_t kind);
/* the structure counts of the handle's current graph (analysed on the host if needed) and the counters of the last solve */
int d2pgo_cholesky_stats(d2pgo_handle *h, d2pgo_cholesky_info *out);
/* parity hook: linearise at the current poses (edges, gravity priors, ARock proximal terms towards the duals' y_r), factor
 * and solve for the given lambda; dx_out[N][D] (0 on fixed poses).  The poses do not move.  Returns 6 (dx_out still written)
 * when a pivot was not positive. */
int d2pgo_debug_exact_step(d2pgo_handle *h, double lambda, double *dx_out, int64_t out_doubles);
/* parity hook: linearise at the current poses as d2pgo_debug_exact_step does and take one step of the PCG solver instead,
 * at most max_it iterations to relative residual tol: dx_out[N][D] (0 on fixed poses), *iters_out the iterations run and
 * *residual_out sqrt(r.r / b.b) of the last update (the CG recurrence; 0 when b = 0).  The poses do not move.  Returns 1 on
 * a null argument, 2 on a small buffer, a negative max_it or a non-finite or negative lambda or tol, 5 with a communicator. */
int d2pgo_debug_pcg_step(d2pgo_handle *h, double lambda, int32_t max_it, double tol, double *dx_out, int64_t out_doubles,
                         int32_t *iters_out, double *residual_out);
/* parity hook: the system the last sparse-Cholesky step on the handle (d2pgo_debug_exact_step or an LM iteration) assembled on
 * the device and factored, copied out (no other device work): diag_out[N][D*D] the damped diagonal block of each pose
 * (row-major, the factored lower triangle mirrored; 0 on fixed poses), b_out[N][D] the right-hand side -g (0 on fixed poses),
 * and the *n_pairs_out distinct pairs of free poses an edge joins, ascending: pair_ab_out[P][2] their pose indices a < b and
 * pair_out[P][D*D] the block H_ab = sum of J_a^T J_b over their edges.  Returns 5 when no step was taken on the handle's
 * current structure, 2 (with *n_pairs_out set) when max_pairs < P. */
int d2pgo_debug_cholesky_system(d2pgo_handle *h, double *diag_out, double *b_out, int32_t max_pairs, int32_t *n_pairs_out,
                                int32_t *pair_ab_out, double *pair_out);
/* the symbolic analysis alone, no device and no handle: n poses, fixed flags (may be NULL), edge ends, D (4 or 6).
 * perm_out[n]: the pose of each block column (the first info->free_poses entries), sn_ptr_out[n + 1]: the first column of
 * each supernode and the end (info->supernodes + 1 entries), sn_parent_out[n]: each supernode's parent, -1 for a root.
 * Returns 1 on a null argument or negative count, 2 on an edge end out of range or another D. */
int d2pgo_cholesky_symbolic(int32_t n, const uint8_t *fixed, int32_t n_edges, const int32_t *ea, const int32_t *eb, int32_t dof,
                            int32_t *perm_out, int32_t *sn_ptr_out, int32_t *sn_parent_out, d2pgo_cholesky_info *info);

/* ---- minimiser of d2pgo_solve and of d2pgo_arock_step's local solve
 *   D2PGO_MINIMIZER_RESTATED  the default: the LM loop above (lambda / 3 on accept, x 4 on reject, one relative-decrease test,
 *                             no time budget; the host reads the cost after every linearisation).  The only kind for PCG and
 *                             for a handle with a communicator.
 *   D2PGO_MINIMIZER_CERES_LM  <- ceres 2.1's TrustRegionMinimizer + LevenbergMarquardtStrategy, as every shipped d2pgo
 *                             configuration runs it: SPARSE_NORMAL_CHOLESKY + LEVENBERG_MARQUARDT with max_solver_time_in_seconds
 *                             = pgo_solver_time (d2pgo/src/d2pgo_node.cpp:190-197; 0.5 or 1.0 s in config/quadcam/*.yaml; the
 *                             test driver d2pgo/test/d2pgo_test.cpp:95-103 uses 0.1 s and 50 iterations), and the ARock local
 *                             solves the same (ARock.cpp:317, d2pgo_node.cpp:202).  With s_k = 1 / (1 + |J_:,k|) from the
 *                             first linearisation (1 without jacobi_scaling), each iteration solves
 *                               (J^T J + diag(mu)) dx = -g,  mu_k = clamp(s_k^2 H_kk, min_lm_diagonal, max_lm_diagonal) / (radius s_k^2)
 *                             over the free poses with the sparse Cholesky (H_kk from the block diagonal; a self loop's cross
 *                             terms are in J^T J, not in H_kk), model m = -(r.J dx + |J dx|^2 / 2), rho = (C - C+) / m; accept
 *                             if rho > min_relative_decrease: radius = min(radius / max(1/3, 1 - (2 rho - 1)^3), max radius),
 *                             decrease factor 2; else radius /= decrease factor, decrease factor *= 2.  A non-positive or
 *                             non-finite pivot, m <= 0 or a non-finite step is an invalid step (rejected; FAILURE after more
 *                             than max_num_consecutive_invalid_steps in a row).  Stops, in this order: gradient (max over the
 *                             free poses' ambient components of |x - x [+] (-g)| <= gradient_tolerance, at the start and after
 *                             every accepted step), iterations (the count of accepted and rejected steps reaches
 *                             max_num_iterations), time (max_solver_time_in_seconds > 0 reached on the device's %globaltimer,
 *                             measured from the solve's first device work, not from the call), parameter (|dx| <=
 *                             parameter_tolerance (|x| + parameter_tolerance), |x| over the free poses' ambient components),
 *                             function (|C - C+| <= function_tolerance C), min radius (radius < min_trust_region_radius after a
 *                             rejection).  A parameter or function stop returns x, not the candidate; that last iteration counts
 *                             as unsuccessful.  ASSUMED (restated from upstream ceres, which is not in the reference tree): the
 *                             Jacobi scale computed once at x0, the gradient test's ambient form, FAILURE after more than 5
 *                             invalid steps, m <= 0 invalid, the parameter and function tests returning x and their order
 *                             (parameter, function, acceptance).  Edges, gravity priors and ARock proximal terms enter as in
 *                             the restated loop.  Needs D2PGO_LINEAR_SPARSE_CHOLESKY and no communicator: otherwise d2pgo_solve
 *                             and d2pgo_arock_step return 5 and do nothing.  The whole solve is one CUDA graph (the iterations
 *                             under a conditional WHILE node, one-thread control kernels deciding on the device) and one host
 *                             synchronisation; it needs a driver for CUDA 12.4 or newer (3 otherwise).
 * d2pgo_report of such a solve: iterations = successful + unsuccessful steps, accepted = successful, converged = (termination
 * type CONVERGENCE), pcg_iterations 0, the costs and device_ms (SolverWrapper.cpp:38-49's mapping of ceres' summary).  The
 * Cholesky counters of d2pgo_cholesky_stats count one factorisation per iteration and no device times. */
enum { D2PGO_MINIMIZER_RESTATED = 0, D2PGO_MINIMIZER_CERES_LM = 1 };
enum { D2PGO_TERMINATION_CONVERGENCE = 0, D2PGO_TERMINATION_NO_CONVERGENCE = 1, D2PGO_TERMINATION_FAILURE = 2 };
enum { D2PGO_STOP_GRADIENT = 1, D2PGO_STOP_PARAMETER = 2, D2PGO_STOP_FUNCTION = 3, D2PGO_STOP_MIN_RADIUS = 4,
       D2PGO_STOP_MAX_ITERATIONS = 5, D2PGO_STOP_TIME = 6, D2PGO_STOP_INVALID_STEPS = 7 };
enum { D2PGO_STEP_ACCEPTED = 0, D2PGO_STEP_REJECTED = 1, D2PGO_STEP_INVALID = 2, D2PGO_STEP_CONVERGED = 3 };

typedef struct d2pgo_ceres_lm_config {   /* ceres::Solver::Options fields; defaults are ceres' */
  int32_t max_num_iterations;            /* 50                                                      */
  int32_t max_num_consecutive_invalid_steps;   /* 5                                                 */
  int32_t jacobi_scaling;                /* 1 (0 or 1)                                              */
  int32_t pad_;
  double max_solver_time_in_seconds;     /* 0 = no budget                                           */
  double initial_trust_region_radius;    /* 1e4                                                     */
  double max_trust_region_radius;        /* 1e16                                                    */
  double min_trust_region_radius;        /* 1e-32                                                   */
  double min_relative_decrease;          /* 1e-3                                                    */
  double min_lm_diagonal, max_lm_diagonal;   /* 1e-6, 1e32                                          */
  double function_tolerance;             /* 1e-6                                                    */
  double gradient_tolerance;             /* 1e-10                                                   */
  double parameter_tolerance;            /* 1e-8                                                    */
} d2pgo_ceres_lm_config;

typedef struct d2pgo_minimizer_summary {   /* the last ceres-LM solve or ARock step                   */
  int32_t termination_type;              /* D2PGO_TERMINATION_*                                     */
  int32_t reason;                        /* D2PGO_STOP_*                                            */
  int32_t successful_steps, unsuccessful_steps;
  int32_t host_syncs;                    /* stream synchronisations of the call: 1, plus 1 for uploading a graph changed
                                            since the last solve and 1 for the Cholesky's first upload of a structure    */
  int32_t pad_;
  double final_radius;
  double elapsed_s;                      /* device seconds on %globaltimer, first device work to the last decision        */
  double initial_cost, final_cost;
} d2pgo_minimizer_summary;

typedef struct d2pgo_minimizer_iteration {   /* one iteration of the trace                               */
  double cost, candidate_cost;           /* C at x, C+ (NaN when no candidate was evaluated)        */
  double model_cost_change;              /* m                                                       */
  double relative_decrease;              /* rho (NaN when no candidate was evaluated)               */
  double step_norm;                      /* |dx|                                                    */
  double radius, decrease_factor;        /* after the iteration's update                            */
  int32_t kind;                          /* D2PGO_STEP_*                                            */
  int32_t pad_;
} d2pgo_minimizer_iteration;

int d2pgo_default_ceres_lm_config(d2pgo_ceres_lm_config *cfg);
/* kind D2PGO_MINIMIZER_RESTATED (cfg ignored) or D2PGO_MINIMIZER_CERES_LM (cfg NULL = the defaults).  Returns 2 on an unknown
 * kind or a config field that is non-finite, negative or inconsistent (min radius <= initial radius <= max radius, radii > 0,
 * 0 < min_lm_diagonal <= max_lm_diagonal, jacobi_scaling 0 or 1); a refusal keeps nothing.  It may change between solves. */
int d2pgo_set_minimizer(d2pgo_handle *h, int32_t kind, const d2pgo_ceres_lm_config *cfg);
/* the report of the last d2pgo_solve / d2pgo_arock_step; 5 when that call did not run the ceres minimiser */
int d2pgo_minimizer_report(d2pgo_handle *h, d2pgo_minimizer_summary *out);
/* parity hook: the per-iteration records of that call (the first 16384 iterations), copied from the device.  *n_out = the
 * records held; returns 2 (with *n_out set) when max < *n_out, 5 as d2pgo_minimizer_report does */
int d2pgo_debug_minimizer_trace(d2pgo_handle *h, int32_t max, int32_t *n_out, d2pgo_minimizer_iteration *out);

/* ---- perturbation chart of the 6-DoF solve (d2pgo's perturb_mode, which d2pgo_node sets for every 6-DoF graph,
 *      d2pgo/src/d2pgo_node.cpp:216)
 *   d2pgo_set_chart     <- PGOState::addFrame's POSE_PERTURB_6D block (d2pgo/src/pgostate.hpp:25-50, BaseParamResInfo.cpp:4-9)
 *   d2pgo_get_poses     <- postPerturbSolve (d2pgo/src/d2pgo.cpp:616-628)
 * In the chart the state of pose f is the Euclidean 6-vector x_f = [p_f, theta_f] (no manifold) and its attitude is
 *     q_f = q_init,f (x) quatfromRotationVector(theta_f),   quatfromRotationVector(t) = [t / 2, 1] (unnormalised) if |t| < 1e-2,
 *                                                           else the exact exponential   (utils.hpp:39-55; [x y z w])
 * The factors are RelPoseFactorPerturbAD (RelPoseFactor.hpp:138-195) and GravityPriorPerturbAD (GravityPrior.hpp:8-46), as
 * written: p_ab = q_a.conjugate() applied to p_b - p_a by Eigen's _transformVector (not a rotation for a non-unit q_a),
 * dq = q_meas (q_a.conjugate() q_b).conjugate(), r = S [p_ab - p_meas ; 2 vec(dq)]; the prior's R_a = q_a.toRotationMatrix()
 * (Eigen's polynomial, exact for unit q only), r = S^T (R_a.row(2) - R_ego.row(2))^T.  The state is kept across solves: each
 * solve starts from the last [p, theta] (postPerturbSolve leaves theta, its reset being commented out).
 *   Entering (chart = D2PGO_CHART_PERTURB): every pose gets x = [p, 0] and q_init = its current attitude, normalised, or for the
 *     listed ids the given q_init4[n][4] (xyzw, normalised here; with q_init4 NULL every pose takes its current attitude and the
 *     ids, which must still be poses of the handle, select nothing).  Entering again restarts from the current attitudes.
 *     D2PGO_CHART_RETRACTION leaves it: the poses become d2pgo_get_poses'.
 *   Fixed poses keep their 6-vector (setStateProperties, d2pgo.cpp:602-610).
 *   d2pgo_set_poses keeps x and q_init of the ids already present (their given pose is ignored); new ids start as on entry.
 *     It still removes every edge and gravity prior, as on any handle.  This is how the node's state grows between solves.
 *   d2pgo_get_poses returns [p, normalise(q_init (x) quatfromRotationVector(theta))] (ASSUMED: Swarm::Pose normalises the
 *     attitude postPerturbSolve gives it; that type is not in the reference tree).  d2pgo_get_perturb returns the raw state.
 *   d2pgo_rot_init runs on those attitudes; afterwards every pose's q_init is its attitude: the rotation-initialised one for the
 *     frames it solves, the current one for the others (recoverRotationLLT, rotation_initialization_base.hpp:360-389); p and
 *     theta keep every bit.
 *   d2pgo_debug_edges / d2pgo_debug_gravity_priors / d2pgo_debug_exact_step / d2pgo_debug_pcg_step report and solve in
 *     [dp, dtheta] of the 6-vector, in the same layouts.
 *   Both minimisers and both linear solvers run in the chart; only the linearisation and the retraction (x <- x + dx) change.
 *   ceres LM: the Jacobi scale is of the 6-vector Jacobian's columns, the gradient test max |x - (x + (-g))| and |x| of the
 *     parameter test run over the free poses' [p, theta] (ASSUMED as for the retraction chart), and the solve's graph is built
 *     again when the chart changes.
 *   ARock (d2pgo_arock_*; ARockPGO runs in perturb mode, ARockPGO.cpp:21-23): the dual coordinates are the state x = [p, theta]
 *     itself (no log map, the ARock q_init of d2pgo_arock_enable is not read), the proximal NormalPrior is
 *     r = diag(sqrt(rho_T) I3, sqrt(rho_theta) I3) (x - y_r) with that diagonal as its constant Jacobian (ARock.cpp:284-291;
 *     d2pgo_debug_arock_terms reports it), and updateDualStates acts on x.  An ARock handle enters or leaves the chart only
 *     while its pose dual table is empty (its duals are coordinates of one chart), and a chart handle refuses the distributed
 *     rotation initialisation (d2pgo_arock_rot_init_step / d2pgo_arock_rot_receive: 5), which d2pgo runs before the perturbation
 *     solve: enter the chart after it, and each q_init is the attitude it left.
 * Not in the chart: 4-DoF handles (d2pgo has no perturbation chart there) and handles with a communicator (the edge-sharded path).
 * Refusals keep nothing of the call and set d2pgo_last_error: 5 on a 4-DoF handle, with a communicator attached (and
 * d2pgo_comm_init returns 5 on a chart handle) or on an ARock handle holding duals; 2 on an unknown chart or id, a non-finite value
 * or a zero q_init (d2pgo_set_poses: a new id's zero quaternion); 1 on a null argument or n < 0.  d2pgo_set_perturb and
 * d2pgo_get_perturb return 5 on a handle not in the chart. */
enum { D2PGO_CHART_RETRACTION = 0, D2PGO_CHART_PERTURB = 1 };
int d2pgo_set_chart(d2pgo_handle *h, int32_t chart, int32_t n, const int64_t *ids, const double *q_init4);
/* x6[n][6] = [p, theta] of the listed poses */
int d2pgo_set_perturb(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *x6);
/* x6_out[n][6] = [p, theta]; q_init4_out[n][4] (may be NULL) their q_init */
int d2pgo_get_perturb(d2pgo_handle *h, int32_t n, const int64_t *ids, double *x6_out, double *q_init4_out);

#ifdef __cplusplus
}
#endif
#endif
