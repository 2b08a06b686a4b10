// d2pgo.cu -- pose-graph optimisation on the GPU (include/d2pgo.h): relative-pose factors, matrix-free block-Jacobi PCG,
// Levenberg-Marquardt outer loop, edge-sharded multi-GPU with one NCCL all-reduce per CG iteration.
//
// Factors: D2Common::RelPoseFactorAD (d2common/include/d2common/solver/RelPoseFactor.hpp:68-135), restated in pgo_edge_eval
// below with analytic exact derivatives in the tangent of the right-multiplicative pose retraction
// (pose_local_parameterization.cpp:13-38).  (The header's hand-differentiated RelPoseFactor :8-66, used when
// pgo_use_autodiff is off, drops q_rel from its rotation blocks -- its Jacobian is exact only for identity relative rotation.)
// And RelPoseFactor4D (:196-238), d2pgo's default 4-DoF configuration, in pgo_edge_eval_4d.  One solver serves both: every
// kernel is a template over an edge policy (PgoEdge6 / PgoEdge4) that fixes the block size D and the retraction.
// Unary gravity priors (GravityPriorPerturbAD, d2pgo's enable_gravity_prior) on 6-DoF poses in pgo_gravity_eval: the kernels
// that sum per-pose terms take a GRAV flag, so the instantiations without priors are the kernels of a graph of edges alone.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/d2pgo.h"
#include "d2ba_math.cuh"

namespace d2ba {
// NCCL through the dlopen'ed entry points of d2ba_host.cu
int nccl_comm_init(void **comm, const uint8_t *unique_id, int rank, int nranks, std::string &err);
int nccl_allreduce_f64(void *comm, double *buf, size_t n, cudaStream_t s);
void nccl_comm_destroy(void *comm);
}  // namespace d2ba
using namespace d2ba;

namespace {

struct PgoScalars {      // device-resident CG state that is not a per-block partial
  double bb;             // |b|^2 of the current linear system
  int done, iters;
};

struct PgoDev {
  int n_pose, n_edge;
  const double *x;        // [N][8] poses the edges are linearised at: [x y z qx qy qz qw 0] (6-DoF) or [x y z yaw 0 0 0 0] (4-DoF)
  const unsigned char *fixed;
  const int *ea, *eb;     // [E] pose indices
  const double *rel;      // [E][8] measurements, same layouts as x
  const double *sinfo;    // [E][D*D] sqrt information, row-major
  double *lin;            // [D + 2 D^2][E] field-major: r(D), J0 (DxD row-major), J1 (DxD)
  double *g, *D;          // [D N], [N][D*D]
  double *Minv;           // [N][D*D]
  double *dx, *r, *z, *p, *Ap;   // [D N]
  double *damp;           // [D N] lambda diag(D) + 1e-12
  double *t;              // [2D][E] per edge: J0^T (J p) (D), J1^T (J p) (D)
  const int *inc_ptr, *inc;   // incidence lists: pose i -> (edge << 1 | side) of this rank's edges, ascending
  double *rz_part, *rr_part;  // [2][nbp] per-block partials, ping-pong on the iteration parity
  double *pAp_part;           // [nbp]
  int nbp;                    // pose blocks of 128
  PgoScalars *s;
};

// gravity priors of this rank (6-DoF only).  A separate, last kernel parameter: read by the GRAV = true instantiations only, it
// leaves the parameter layout of the edge-only kernels as it was.
struct PgoPriorDev {
  int n_prior;
  const int *pose;            // [G] pose index of each prior
  const int *prior_of;        // [N] the prior of each pose, -1 = none
  const double *u, *S;        // [G][3] u_ego = R(q_ego)^T e3, [G][9] S row-major
  double *lin;                // [12][G] field-major: r(3), J_theta (3x3 row-major)
};

// RelPoseFactorAD (RelPoseFactor.hpp:68-135; the reference's default 6-DoF factor, pgo_use_autodiff = true in
// d2pgo/src/d2pgo_config.h:52): r = S [ q_a^-1 (p_b - p_a) - p_meas ; 2 vec(q_meas (q_a^-1 q_b)^-1) ] with the full 6x6 S.
// The reference differentiates it with ceres autodiff on the EigenQuaternionManifold; here the exact derivatives are analytic,
// in the tangent of the right-multiplicative pose retraction (the minimiser does not depend on the manifold chart):
//   d p_ab / d dp_a = -Ra^T,  d p_ab / d dth_a = [p_ab]x,  d p_ab / d dp_b = Ra^T,
//   d 2vec(dq) / d dth_a = (w I + [v]x) of dq,   d 2vec(dq) / d dth_b = -(Qleft(q_meas) Qright(q_b^-1 q_a))_3.
D2BA_DEV void pgo_edge_eval(const double *p0, const double *p1, const double *rel, const double *S, double *r, double *J0, double *J1) {
  const Q4 q0 = qload(p0 + 3), q1 = qload(p1 + 3), qm = qload(rel + 3);
  const Q4 q0i = Q4{-q0.x, -q0.y, -q0.z, q0.w}, q1i = Q4{-q1.x, -q1.y, -q1.z, q1.w};   // conjugates (:83)
  double R0i[9];
  q2R(q0i, R0i);
  const double dt[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
  double pab[3];
  mv3(R0i, dt, pab);                                  // q_a_inverse * (p_b - p_a) (:87)
  const Q4 X = qmul(q1i, q0);                         // (q_a^-1 q_b)^-1
  const Q4 dq = qmul(qm, X);                          // q_measured * q_ab_estimated.conjugate() (:90-91)
  const double raw[6] = {pab[0] - rel[0], pab[1] - rel[1], pab[2] - rel[2], 2.0 * dq.x, 2.0 * dq.y, 2.0 * dq.z};
  for (int i = 0; i < 6; i++) { double t = 0; for (int k = 0; k < 6; k++) t += S[i * 6 + k] * raw[k]; r[i] = t; }   // applyOnTheLeft (:104)
  if (!J0) return;
  double A0[36], A1[36];
  for (int i = 0; i < 36; i++) { A0[i] = 0.0; A1[i] = 0.0; }
  const double Sk[9] = {0, -pab[2], pab[1], pab[2], 0, -pab[0], -pab[1], pab[0], 0};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { A0[i * 6 + j] = -R0i[i * 3 + j]; A1[i * 6 + j] = R0i[i * 3 + j]; A0[i * 6 + 3 + j] = Sk[i * 3 + j]; }
  const double L[9] = {dq.w, -dq.z, dq.y, dq.z, dq.w, -dq.x, -dq.y, dq.x, dq.w};   // w I + [v]x of dq
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) A0[(3 + i) * 6 + 3 + j] = L[i * 3 + j];
  const double Lm[9] = {qm.w, -qm.z, qm.y, qm.z, qm.w, -qm.x, -qm.y, qm.x, qm.w};  // w I + [v]x of q_meas
  const double Rx[9] = {X.w, X.z, -X.y, -X.z, X.w, X.x, X.y, -X.x, X.w};            // w I - [v]x of X
  double P[9];
  mm3(Lm, Rx, P);
  const double vm[3] = {qm.x, qm.y, qm.z}, vx[3] = {X.x, X.y, X.z};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) A1[(3 + i) * 6 + 3 + j] = -(P[i * 3 + j] - vm[i] * vx[j]);
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
    double t0 = 0, t1 = 0;
    for (int k = 0; k < 6; k++) { t0 += S[i * 6 + k] * A0[k * 6 + j]; t1 += S[i * 6 + k] * A1[k * 6 + j]; }
    J0[i * 6 + j] = t0; J1[i * 6 + j] = t1;
  }
}

// Utility::NormalizeAngle (d2common/include/d2common/utils.hpp:251-257): a - 2 pi floor((a + pi) / 2 pi), in [-pi, pi)
D2BA_DEV double pgo_normalize_angle(double a) { return a - 2.0 * M_PI * floor((a + M_PI) / (2.0 * M_PI)); }

// RelPoseFactor4D (RelPoseFactor.hpp:216-227 + Utility::poseError4D, utils.hpp:240-280; d2pgo's default pgo_pose_dof =
// PGO_POSE_4D): poses [x y z yaw], v = p_b - p_a,
//   r = S [ p_meas - Rz(-yaw_a) v ; N(yaw_meas - N(yaw_b - yaw_a)) ]   with the full 4x4 S, and the exact Jacobians
//   d/d p_a = S [Rz(-yaw_a); 0],  d/d yaw_a = S [Rz'(-yaw_a) v; 1],  d/d p_b = S [-Rz(-yaw_a); 0],  d/d yaw_b = S [0; -1]
// (PosAngleManifold's tangent is the 4-vector itself).  The CPU oracle states the same lines (edge_eval_4d).
D2BA_DEV void pgo_edge_eval_4d(const double *pa, const double *pb, const double *rel, const double *S, double *r, double *J0, double *J1) {
  double s, c;
  sincos(-pa[3], &s, &c);
  const double v[3] = {pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]};
  const double raw[4] = {rel[0] - (c * v[0] - s * v[1]), rel[1] - (s * v[0] + c * v[1]), rel[2] - v[2],
                         pgo_normalize_angle(rel[3] - pgo_normalize_angle(pb[3] - pa[3]))};
  for (int i = 0; i < 4; i++) { double t = 0; for (int k = 0; k < 4; k++) t += S[i * 4 + k] * raw[k]; r[i] = t; }
  if (!J0) return;
  // A0 = [Rz | Rz' v ; 0 0 0 1], A1 = [-Rz | 0 ; 0 0 0 -1]; Rz' = d Rz(t) / dt at t = -yaw_a
  const double A0[16] = {c, -s, 0.0, -s * v[0] - c * v[1],
                         s, c, 0.0, c * v[0] - s * v[1],
                         0.0, 0.0, 1.0, 0.0,
                         0.0, 0.0, 0.0, 1.0};
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double t0 = 0;
    for (int k = 0; k < 4; k++) t0 += S[i * 4 + k] * A0[k * 4 + j];
    J0[i * 4 + j] = t0;
    J1[i * 4 + j] = j < 3 ? -t0 : -S[i * 4 + 3];   // S A1: the position columns are those of S A0 negated
  }
}

// Edge-evaluation policies: block size D of the tangent, stored pose width NX (of the 8 doubles per pose) and the retraction.
struct PgoEdge6 {   // RelPoseFactorAD on [x y z qx qy qz qw], PoseLocalParameterization::Plus
  static constexpr int D = 6, NX = 7;
  D2BA_DEV static void eval(const double *p0, const double *p1, const double *rel, const double *S, double *r, double *J0, double *J1) { pgo_edge_eval(p0, p1, rel, S, r, J0, J1); }
  D2BA_DEV static void plus(const double *x, const double *dx, double *o) { pose_plus(x, dx, o); }
};
struct PgoEdge4 {   // RelPoseFactor4D on [x y z yaw], PosAngleManifold::Plus (angle_manifold.h:39-68): x + dx, yaw normalised
  static constexpr int D = 4, NX = 4;
  D2BA_DEV static void eval(const double *p0, const double *p1, const double *rel, const double *S, double *r, double *J0, double *J1) { pgo_edge_eval_4d(p0, p1, rel, S, r, J0, J1); }
  D2BA_DEV static void plus(const double *x, const double *dx, double *o) {
    for (int k = 0; k < 3; k++) o[k] = x[k] + dx[k];
    o[3] = pgo_normalize_angle(x[3] + dx[3]);
  }
};

// GravityPriorPerturbAD (GravityPrior.hpp:8-46, added per frame by D2PGO::setupGravityPriorFactors, d2pgo.cpp:530-559):
// u = R(q)^T e3 (the third row of R), r = S^T (u - u_ego) -- the reference forms the row R.row(2) - R_ego.row(2) and applies
// S on the right.  In the tangent of the right-multiplicative retraction: dr/d dtheta = S^T [u]x, dr/d dp = 0 (rank 2: yaw
// about gravity stays free).  The reference's chart q0 (x) quatfromRotationVector(theta) has the same value and derivative at
// theta = 0; inside |theta| < 1e-2 it uses the unnormalised [1, theta/2], which this evaluation at the exact pose does not.
D2BA_DEV void pgo_gravity_eval(const double *x, const double *ue, const double *S, double *r, double *J) {
  double R[9];
  q2R(qload(x + 3), R);
  const double u[3] = {R[6], R[7], R[8]};
  const double du[3] = {u[0] - ue[0], u[1] - ue[1], u[2] - ue[2]};
  for (int i = 0; i < 3; i++) r[i] = S[i] * du[0] + S[3 + i] * du[1] + S[6 + i] * du[2];
  if (!J) return;
  const double K[9] = {0.0, -u[2], u[1], u[2], 0.0, -u[0], -u[1], u[0], 0.0};   // [u]x
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[i * 3 + j] = S[i] * K[j] + S[3 + i] * K[3 + j] + S[6 + i] * K[6 + j];
}

// Fixed-order sum of n per-block partials, the same value in every thread of every block (so that all blocks -- and all
// ranks, which hold identical vectors -- take the same branch without a single-thread "decide" kernel in between).
D2BA_DEV double total_of(const double *part, int n, double *red) {
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = 0.0;
    for (int i = threadIdx.x; i < n; i += 32) v += part[i];
    v = warp_sum(v);
    if (threadIdx.x == 0) red[39] = v;
  }
  __syncthreads();
  return red[39];
}

// linearise every local edge at d.x: lin records [r | J0 | J1] and per-block cost partials (summed in fixed order by k_pgo_sum)
template <class P>
__global__ void __launch_bounds__(128) k_pgo_lin(PgoDev d, double *cost_part, int want_jac) {
  constexpr int D = P::D, DD = D * D;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (e < d.n_edge) {
    const int a = d.ea[e], b = d.eb[e];
    double r[D], J0[DD], J1[DD];
    P::eval(d.x + (size_t)a * 8, d.x + (size_t)b * 8, d.rel + (size_t)e * 8, d.sinfo + (size_t)e * DD, r, want_jac ? J0 : nullptr, J1);
    for (int k = 0; k < D; k++) c += 0.5 * r[k] * r[k];
    if (want_jac) {
      double *o = d.lin + e;   // field-major [D + 2 D^2][E]: consecutive edges (threads) touch consecutive addresses
      const size_t E = (size_t)d.n_edge;
      for (int k = 0; k < D; k++) o[k * E] = r[k];
      for (int k = 0; k < DD; k++) { o[(D + k) * E] = J0[k]; o[(D + DD + k) * E] = J1[k]; }
    }
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}
// linearise every local gravity prior at d.x: glin records [r | J_theta]; cost partials go after the edges' (k_pgo_sum)
__global__ void __launch_bounds__(128) k_pgo_prior_lin(PgoDev d, double *cost_part, int want_jac, PgoPriorDev pr) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (k < pr.n_prior) {
    double r[3], J[9];
    pgo_gravity_eval(d.x + (size_t)pr.pose[k] * 8, pr.u + (size_t)k * 3, pr.S + (size_t)k * 9, r, J);   // J always: keeps r, J in registers
    for (int a = 0; a < 3; a++) c += 0.5 * r[a] * r[a];
    if (want_jac) {
      double *o = pr.lin + k;
      const size_t G = (size_t)pr.n_prior;
      for (int a = 0; a < 3; a++) o[a * G] = r[a];
      for (int a = 0; a < 9; a++) o[(3 + a) * G] = J[a];
    }
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}

// pose i's gravity prior, after its edges: g += J^T r, D += J^T J on the rotation block (D = 6 only)
template <int D>
D2BA_DEV void prior_gD(const PgoPriorDev &pr, int i, double *gi, double *Di) {
  const int k = pr.prior_of[i];
  if (k < 0) return;
  const size_t G = (size_t)pr.n_prior;
  const double *o = pr.lin + k;
  for (int a = 0; a < 3; a++) {
    const double ra = o[a * G];
    double row[3];
    for (int b = 0; b < 3; b++) { row[b] = o[(3 + a * 3 + b) * G]; gi[3 + b] += row[b] * ra; }
    for (int b = 0; b < 3; b++) for (int c = 0; c < 3; c++) Di[(3 + b) * D + 3 + c] += row[b] * row[c];
  }
}

// pose i's gravity prior in a CG product: y += J^T (J p) on the rotation block
template <int D>
D2BA_DEV void prior_Ap(const PgoPriorDev &pr, int i, const double *p, double *y) {
  const int k = pr.prior_of[i];
  if (k < 0) return;
  const size_t G = (size_t)pr.n_prior;
  const double *J = pr.lin + (size_t)3 * G + k;
  for (int a = 0; a < 3; a++) {
    double j[3], t = 0.0;
    for (int b = 0; b < 3; b++) { j[b] = J[(size_t)(a * 3 + b) * G]; t += j[b] * p[3 + b]; }
    for (int b = 0; b < 3; b++) y[3 + b] += j[b] * t;
  }
}

__global__ void k_pgo_sum(const double *part, int n, double *out) {
  __shared__ double red[40];
  const double v = total_of(part, n, red);
  if (threadIdx.x == 0) out[0] = v;
}

// gradient g_i = sum J^T r and block diagonal D_i = sum J^T J over the edges incident to pose i, in the fixed order of the
// incidence list (no atomics: bitwise reproducible); with GRAV, the pose's gravity prior after its edges
template <class P, bool GRAV>
__global__ void __launch_bounds__(128) k_pgo_gD(PgoDev d, double *g, double *Dg, PgoPriorDev pr) {
  constexpr int D = P::D, DD = D * D;
  static_assert(!GRAV || D == 6, "gravity priors act on 6-DoF poses");
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n_pose) return;
  double gi[D], Di[DD];
  for (int k = 0; k < D; k++) gi[k] = 0.0;
  for (int k = 0; k < DD; k++) Di[k] = 0.0;
  if (!d.fixed[i]) {
    for (int q = d.inc_ptr[i]; q < d.inc_ptr[i + 1]; q++) {
      const int c = d.inc[q];
      const size_t E = (size_t)d.n_edge;
      const double *o = d.lin + (c >> 1), *J = o + (size_t)(D + DD * (c & 1)) * E;
      for (int k = 0; k < D; k++) {
        const double rk = o[k * E];
        double row[D];
        for (int a = 0; a < D; a++) { row[a] = J[(size_t)(k * D + a) * E]; gi[a] += row[a] * rk; }
        for (int a = 0; a < D; a++) for (int b = 0; b < D; b++) Di[a * D + b] += row[a] * row[b];
      }
    }
    if constexpr (GRAV) prior_gD<D>(pr, i, gi, Di);
  }
  for (int k = 0; k < D; k++) g[(size_t)i * D + k] = gi[k];
  for (int k = 0; k < DD; k++) Dg[(size_t)i * DD + k] = Di[k];
}

// block-Jacobi preconditioner: Minv = (D + lambda diag(D))^-1 per free pose (DxD Cholesky, one thread per pose); also the
// damping diagonal lambda diag(D) + 1e-12 the products add
template <class P>
__global__ void k_pgo_precond(PgoDev d, const double *Dg, double lambda) {
  constexpr int D = P::D, DD = D * D;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n_pose) return;
  double *M = d.Minv + (size_t)i * DD;
  if (d.fixed[i]) { for (int k = 0; k < DD; k++) M[k] = 0.0; for (int k = 0; k < D; k++) d.damp[(size_t)i * D + k] = 0.0; return; }
  double A[DD], Li[DD];
  for (int k = 0; k < DD; k++) A[k] = Dg[(size_t)i * DD + k];
  for (int k = 0; k < D; k++) { const double dk = lambda * A[k * (D + 1)] + 1e-12; d.damp[(size_t)i * D + k] = dk; A[k * (D + 1)] += dk; }
  for (int j = 0; j < D; j++) {   // Cholesky, lower
    double s = A[j * D + j];
    for (int k = 0; k < j; k++) s -= A[j * D + k] * A[j * D + k];
    s = sqrt(s > 0.0 ? s : 1e-300);
    A[j * D + j] = s;
    for (int r = j + 1; r < D; r++) { double t = A[r * D + j]; for (int k = 0; k < j; k++) t -= A[r * D + k] * A[j * D + k]; A[r * D + j] = t / s; }
  }
  for (int c = 0; c < D; c++) {   // L^-1 column by column
    for (int r = 0; r < D; r++) {
      double t = r == c ? 1.0 : 0.0;
      for (int k = 0; k < r; k++) t -= A[r * D + k] * Li[k * D + c];
      Li[r * D + c] = t / A[r * D + r];
    }
  }
  for (int r = 0; r < D; r++) for (int c = 0; c < D; c++) { double t = 0; for (int k = 0; k < D; k++) t += Li[k * D + r] * Li[k * D + c]; M[r * D + c] = t; }
}

// ---- conjugate gradients.  One iteration = three kernels (the three grid-wide dependencies of CG):
//   k_pgo_cg_edge : per edge J0^T t, J1^T t with t = J0 p_a + J1 p_b, p = z + beta p_old formed on the fly   (needs rz of the last update)
//   k_pgo_cg_pose : stores p, Ap_i = sum over incident edges (+ damping), partials of p.Ap               (needs every edge)
//   k_pgo_cg_step : alpha = rz / pAp; dx += alpha p; r -= alpha Ap; z = Minv r; partials of r.z, r.r   (needs p.Ap)
// Scalars live as per-block partials summed in fixed order by every block (total_of); rz / rr ping-pong on the iteration
// parity `par`.  Once converged the sticky flag s->done turns the remaining launches of a graph into no-ops.
struct CgView { double rz_prev, rz_cur, rr_cur; bool done, first; };
D2BA_DEV CgView cg_view(const PgoDev &d, int par, double tol2, double *red) {
  CgView v;
  const PgoScalars *s = d.s;
  v.first = s->iters == 0;
  v.rz_cur = total_of(d.rz_part + (size_t)(par ^ 1) * d.nbp, d.nbp, red);
  v.rr_cur = total_of(d.rr_part + (size_t)(par ^ 1) * d.nbp, d.nbp, red);
  v.rz_prev = v.first ? 1.0 : total_of(d.rz_part + (size_t)par * d.nbp, d.nbp, red);
  v.done = s->done || !(v.rr_cur > tol2 * s->bb) || !(v.rz_cur > 0.0) || !isfinite(v.rz_cur);
  return v;
}
template <int D>
D2BA_DEV void cg_p_new(const PgoDev &d, int i, double beta, double *p) {
  for (int k = 0; k < D; k++) p[k] = d.z[(size_t)i * D + k] + beta * d.p[(size_t)i * D + k];   // p holds 0 before the first iteration
}

template <class P>
__global__ void __launch_bounds__(128) k_pgo_cg_edge(PgoDev d, int par, double tol2) {
  constexpr int D = P::D, DD = D * D;
  __shared__ double red[40];
  const CgView v = cg_view(d, par, tol2, red);
  if (v.done) return;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= d.n_edge) return;
  const double beta = v.first ? 0.0 : v.rz_cur / v.rz_prev;
  const int a = d.ea[e], b = d.eb[e];
  const size_t E = (size_t)d.n_edge;
  const double *J0 = d.lin + D * E + e, *J1 = J0 + DD * E;
  double pa[D], pb[D], ya[D], yb[D];
  for (int q = 0; q < D; q++) { ya[q] = 0.0; yb[q] = 0.0; }
  cg_p_new<D>(d, a, beta, pa); cg_p_new<D>(d, b, beta, pb);
  // t = J0 pa + J1 pb, then this edge's two contributions J0^T t, J1^T t (the Jacobians are read once, coalesced; the
  // per-pose kernel only sums D numbers per incident edge)
  for (int k = 0; k < D; k++) {
    double j0[D], j1[D], tk = 0;
    for (int q = 0; q < D; q++) { j0[q] = J0[(size_t)(k * D + q) * E]; j1[q] = J1[(size_t)(k * D + q) * E]; tk += j0[q] * pa[q] + j1[q] * pb[q]; }
    for (int q = 0; q < D; q++) { ya[q] += j0[q] * tk; yb[q] += j1[q] * tk; }
  }
  for (int q = 0; q < D; q++) { d.t[(size_t)q * E + e] = ya[q]; d.t[(size_t)(D + q) * E + e] = yb[q]; }
}

// LOCAL: this rank's edges only, no damping / p.Ap yet (the all-reduce of Ap comes first; k_pgo_cg_pAp follows).
// GRAV: the pose's gravity prior after its edges.
template <class P, bool LOCAL, bool GRAV>
__global__ void __launch_bounds__(128) k_pgo_cg_pose(PgoDev d, int par, double tol2, PgoPriorDev pr) {
  constexpr int D = P::D;
  static_assert(!GRAV || D == 6, "gravity priors act on 6-DoF poses");
  __shared__ double red[40];
  const CgView v = cg_view(d, par, tol2, red);
  if (v.done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (i < d.n_pose) {
    const double beta = v.first ? 0.0 : v.rz_cur / v.rz_prev;
    double p[D], y[D];
    for (int k = 0; k < D; k++) y[k] = 0.0;
    cg_p_new<D>(d, i, beta, p);
    if (!d.fixed[i]) {
      for (int q = d.inc_ptr[i]; q < d.inc_ptr[i + 1]; q++) {
        const int c = d.inc[q];
        const size_t E = (size_t)d.n_edge;
        const double *t = d.t + (size_t)(D * (c & 1)) * E + (c >> 1);
        for (int a = 0; a < D; a++) y[a] += t[a * E];
      }
      if constexpr (GRAV) prior_Ap<D>(pr, i, p, y);
    }
    for (int k = 0; k < D; k++) {
      d.p[(size_t)i * D + k] = p[k];
      if (!LOCAL) { y[k] += d.damp[(size_t)i * D + k] * p[k]; s += p[k] * y[k]; }
      d.Ap[(size_t)i * D + k] = y[k];
    }
  }
  if (!LOCAL) { s = block_sum(s, red); if (threadIdx.x == 0) d.pAp_part[blockIdx.x] = s; }
}

template <class P>
__global__ void __launch_bounds__(128) k_pgo_cg_pAp(PgoDev d, int par, double tol2) {   // multi-rank: after the all-reduce of Ap
  constexpr int D = P::D;
  __shared__ double red[40];
  const CgView v = cg_view(d, par, tol2, red);
  if (v.done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (i < d.n_pose)
    for (int k = 0; k < D; k++) {
      const double pk = d.p[(size_t)i * D + k], y = d.Ap[(size_t)i * D + k] + d.damp[(size_t)i * D + k] * pk;
      d.Ap[(size_t)i * D + k] = y; s += pk * y;
    }
  s = block_sum(s, red);
  if (threadIdx.x == 0) d.pAp_part[blockIdx.x] = s;
}

template <class P>
__global__ void __launch_bounds__(128) k_pgo_cg_step(PgoDev d, int par, double tol2) {
  constexpr int D = P::D, DD = D * D;
  __shared__ double red[40];
  const CgView v = cg_view(d, par, tol2, red);
  if (v.done) { if (blockIdx.x == 0 && threadIdx.x == 0) d.s->done = 1; return; }
  const double pAp = total_of(d.pAp_part, d.nbp, red);
  const double alpha = pAp > 0.0 ? v.rz_cur / pAp : 0.0;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double rz = 0, rr = 0;
  if (i < d.n_pose && !d.fixed[i]) {
    double r[D];
    for (int k = 0; k < D; k++) {
      d.dx[(size_t)i * D + k] += alpha * d.p[(size_t)i * D + k];
      r[k] = d.r[(size_t)i * D + k] - alpha * d.Ap[(size_t)i * D + k];
      d.r[(size_t)i * D + k] = r[k];
    }
    const double *M = d.Minv + (size_t)i * DD;
    for (int k = 0; k < D; k++) { double t = 0; for (int q = 0; q < D; q++) t += M[k * D + q] * r[q]; d.z[(size_t)i * D + k] = t; rz += r[k] * t; rr += r[k] * r[k]; }
  }
  rz = block_sum(rz, red); rr = block_sum(rr, red);
  if (threadIdx.x == 0) {
    d.rz_part[(size_t)par * d.nbp + blockIdx.x] = rz; d.rr_part[(size_t)par * d.nbp + blockIdx.x] = rr;
    if (blockIdx.x == 0) d.s->iters = d.s->iters + 1;   // read by the next kernel, not by this one's other blocks (cg_view ran before)
  }
}

// CG start: dx = 0, r = -g, z = Minv r, p = 0 (the first k_pgo_cg_edge forms p = z); partials into the parity-1 slots
template <class P>
__global__ void __launch_bounds__(128) k_pgo_cg_init(PgoDev d, const double *g) {
  constexpr int D = P::D, DD = D * D;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double rz = 0, rr = 0;
  if (i < d.n_pose) {
    double r[D], z[D];
    for (int k = 0; k < D; k++) r[k] = d.fixed[i] ? 0.0 : -g[(size_t)i * D + k];
    const double *M = d.Minv + (size_t)i * DD;
    for (int k = 0; k < D; k++) { double t = 0; for (int q = 0; q < D; q++) t += M[k * D + q] * r[q]; z[k] = t; }
    for (int k = 0; k < D; k++) {
      d.dx[(size_t)i * D + k] = 0.0; d.r[(size_t)i * D + k] = r[k]; d.z[(size_t)i * D + k] = z[k]; d.p[(size_t)i * D + k] = 0.0;
      rz += r[k] * z[k]; rr += r[k] * r[k];
    }
  }
  rz = block_sum(rz, red); rr = block_sum(rr, red);
  if (threadIdx.x == 0) { d.rz_part[(size_t)d.nbp + blockIdx.x] = rz; d.rr_part[(size_t)d.nbp + blockIdx.x] = rr; }
}
__global__ void k_pgo_cg_init2(PgoDev d) {   // |b|^2 and the counters
  __shared__ double red[40];
  const double bb = total_of(d.rr_part + d.nbp, d.nbp, red);
  if (threadIdx.x == 0) { d.s->bb = bb; d.s->done = 0; d.s->iters = 0; }
}

// candidate poses: x_out = x (+) dx   (PoseLocalParameterization::Plus / PosAngleManifold::Plus); unused slots zero
template <class P>
__global__ void k_pgo_retract(PgoDev d, double *x_out) {
  constexpr int NX = P::NX;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n_pose) return;
  const double *x = d.x + (size_t)i * 8;
  double o[NX];
  if (d.fixed[i]) { for (int k = 0; k < NX; k++) o[k] = x[k]; }
  else P::plus(x, d.dx + (size_t)i * P::D, o);
  for (int k = 0; k < NX; k++) x_out[(size_t)i * 8 + k] = o[k];
  for (int k = NX; k < 8; k++) x_out[(size_t)i * 8 + k] = 0.0;
}

template <typename T> struct Buf {
  T *p = nullptr; size_t n = 0;
  cudaError_t alloc(size_t c) { if (c <= n && p) return cudaSuccess; if (p) cudaFree(p); p = nullptr; n = 0; cudaError_t e = cudaMalloc(&p, (c ? c : 1) * sizeof(T)); if (e == cudaSuccess) n = c; return e; }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

// ---- PCM: pairwise-consistency maximisation over the loop closures (SwarmLocalOutlierRejection, non-incremental, redundant;
// d2pgo/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:46-303).  Loops are grouped by the unordered pair of drones;
// a group's loops occupy consecutive slots in input order.  Per group: a bit-packed adjacency [L][W = ceil(L/32)] words,
// bit (i, j) = smd(edge1 = max(i, j), edge2 = min(i, j)) < thres, then FMC maxCliqueHeu on it; inlier = in the clique.
constexpr int kPcmMaxGroup = 32768;   // 128 MB of adjacency bits
constexpr int kPcmWarps = 8;          // warps of a k_pcm_clique CTA = seeds examined per round

struct PcmDev {
  const int *g_loop;          // [G+1] slot offsets of the groups
  const long long *g_word;    // [G+1] adjacency word offsets (sum of L W)
  const long long *g_smd;     // [G+1] offsets of the tested pairs (sum of L (L-1) / 2)
  const int *fa, *fb;         // [n] frame index of the loop's two keyframes, by slot
  const unsigned char *flip;  // [n] drone ids in the opposite order to the other loops of the group with flip = 0
  const double *rel;          // [n][8] measured T_a^-1 T_b [t, q xyzw], by slot
  const double *cov;          // [n][21] loop covariance (S^T S)^-1, packed lower triangle, by slot
  const double *ego;          // [F][8] ego poses
  const double *path;         // [F] path length of the frame's drone from its first keyframe
  unsigned *adj; int *deg; double *smd;
  int is4; double thr, pos_cov, yaw_cov;
};

struct Pose7 { double t[3]; Q4 q; };
D2BA_DEV Q4 qnormalized(const Q4 &q) { const double s = 1.0 / sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w); return Q4{q.x * s, q.y * s, q.z * s, q.w * s}; }
D2BA_DEV Pose7 p7_load(const double *p) { return Pose7{{p[0], p[1], p[2]}, qnormalized(qload(p + 3))}; }
D2BA_DEV Pose7 p7_mul(const Pose7 &a, const Pose7 &b) {   // a * b (Swarm::Pose composition; attitude normalised as its constructor does)
  double R[9], v[3];
  q2R(a.q, R); mv3(R, b.t, v);
  return Pose7{{v[0] + a.t[0], v[1] + a.t[1], v[2] + a.t[2]}, qnormalized(qmul(a.q, b.q))};
}
D2BA_DEV Pose7 p7_inv(const Pose7 &a) {
  const Q4 qi = qinv(a.q);
  double R[9], v[3];
  q2R(qi, R); mv3(R, a.t, v);
  return Pose7{{-v[0], -v[1], -v[2]}, qnormalized(qi)};
}
D2BA_DEV double quat_yaw(const Q4 &q) { return atan2(2.0 * (q.w * q.z + q.x * q.y), 1.0 - 2.0 * (q.y * q.y + q.z * q.z)); }

// ego motion from frame f to frame g of one drone: DeltaPose(ego_f, ego_g[, yaw only]) and the diagonal of d2pgo's ego-motion
// covariance (d2pgo.cpp:482-493) at the path length between them (ASSUMED DroneTrajectory::get_relative_pose_by_frame_id)
D2BA_DEV Pose7 pcm_odom(const PcmDev &d, int f, int g, double *cp, double *cr) {
  const Pose7 a = p7_load(d.ego + (size_t)f * 8), b = p7_load(d.ego + (size_t)g * 8);
  const double len = fabs(d.path[g] - d.path[f]);
  *cp = d.pos_cov * len + 0.5 * d.yaw_cov * len * len;
  *cr = d.yaw_cov * len;
  if (!d.is4) return p7_mul(p7_inv(a), b);
  const double ya = quat_yaw(a.q), dy = quat_yaw(b.q) - ya;
  double s, c, sh, ch;
  sincos(ya, &s, &c); sincos(0.5 * dy, &sh, &ch);
  const double v[3] = {b.t[0] - a.t[0], b.t[1] - a.t[1], b.t[2] - a.t[2]};
  return Pose7{{c * v[0] + s * v[1], -s * v[0] + c * v[1], v[2]}, qnormalized(Q4{0.0, 0.0, sh, ch})};
}

// squared Mahalanobis distance of the loop pair (edge1 = slot e1, edge2 = slot e2; swarm_outlier_rejection.cpp:141-199)
D2BA_DEV double pcm_smd(const PcmDev &d, int e1, int e2) {
  const bool same = d.flip[e1] == d.flip[e2];   // same_robot_pair 1; otherwise 2
  Pose7 p2 = p7_load(d.rel + (size_t)e2 * 8);
  if (!same) p2 = p7_inv(p2);
  double ca_p, ca_r, cb_p, cb_r;
  const Pose7 oa = pcm_odom(d, d.fa[e1], same ? d.fa[e2] : d.fb[e2], &ca_p, &ca_r);
  const Pose7 ob = pcm_odom(d, d.fb[e1], same ? d.fb[e2] : d.fa[e2], &cb_p, &cb_r);
  const Pose7 err = p7_mul(p7_mul(p7_mul(oa, p2), p7_inv(ob)), p7_inv(p7_load(d.rel + (size_t)e1 * 8)));
  // log_map (ASSUMED = tangentSpace: [t ; angle-axis], angle = 2 atan2(|v|, |w|), sign of w)
  double v[6] = {err.t[0], err.t[1], err.t[2], 0.0, 0.0, 0.0};
  const double n = sqrt(err.q.x * err.q.x + err.q.y * err.q.y + err.q.z * err.q.z);
  if (n > 0.0) {
    const double k = 2.0 * atan2(n, fabs(err.q.w)) * (err.q.w < 0.0 ? -1.0 : 1.0) / n;
    v[3] = k * err.q.x; v[4] = k * err.q.y; v[5] = k * err.q.z;
  }
  // Sigma = (cov_1 + cov_2) + (cov(odom_a) + cov(odom_b)), then v^T Sigma^-1 v by Cholesky (packed lower triangle)
  double A[21];
  const double *c1 = d.cov + (size_t)e1 * 21, *c2 = d.cov + (size_t)e2 * 21;
  for (int k = 0; k < 21; k++) A[k] = c1[k] + c2[k];
  for (int k = 0; k < 6; k++) A[k * (k + 3) / 2] += k < 3 ? ca_p + cb_p : ca_r + cb_r;
  double y[6], s = 0.0;
  for (int j = 0; j < 6; j++) {
    double t = A[j * (j + 1) / 2 + j];
    for (int k = 0; k < j; k++) t -= A[j * (j + 1) / 2 + k] * A[j * (j + 1) / 2 + k];
    const double l = sqrt(t);
    A[j * (j + 1) / 2 + j] = l;
    for (int r = j + 1; r < 6; r++) {
      double u = A[r * (r + 1) / 2 + j];
      for (int k = 0; k < j; k++) u -= A[r * (r + 1) / 2 + k] * A[j * (j + 1) / 2 + k];
      A[r * (r + 1) / 2 + j] = u / l;
    }
    double w = v[j];
    for (int k = 0; k < j; k++) w -= A[j * (j + 1) / 2 + k] * y[k];
    y[j] = w / l;
    s += y[j] * y[j];
  }
  return s;
}

// per drone (one warp each): path length from its first keyframe, in trajectory order, by a fixed-order warp scan
__global__ void k_pcm_path(int n_drones, const int *traj_ptr, const int *traj, const double *ego, double *path) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_drones) return;
  const int b = traj_ptr[w], n = traj_ptr[w + 1] - b;
  double carry = 0.0;
  for (int base = 0; base < n; base += 32) {
    const int k = base + lane;
    double x = 0.0;
    if (k > 0 && k < n) {
      const double *p = ego + (size_t)traj[b + k] * 8, *q = ego + (size_t)traj[b + k - 1] * 8;
      const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
      x = sqrt(dx * dx + dy * dy + dz * dz);
    }
    for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += u; }
    if (k < n) path[traj[b + k]] = carry + x;
    carry += __shfl_sync(0xffffffffu, x, 31);
  }
}

// per loop slot: measurement in slot order and covariance = (S^T S)^-1 (ASSUMED LoopEdge::getCovariance)
__global__ void k_pcm_loop(int n, const int *src, const double *rel7, const double *sqrt36, double *rel, double *cov) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const size_t s = (size_t)src[e];
  for (int k = 0; k < 7; k++) rel[(size_t)e * 8 + k] = rel7[s * 7 + k];
  rel[(size_t)e * 8 + 7] = 0.0;
  const double *S = sqrt36 + s * 36;
  double A[36], Li[36];
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { double t = 0; for (int k = 0; k < 6; k++) t += S[k * 6 + i] * S[k * 6 + j]; A[i * 6 + j] = t; }
  for (int j = 0; j < 6; j++) {   // A = L L^T
    double t = A[j * 7];
    for (int k = 0; k < j; k++) t -= A[j * 6 + k] * A[j * 6 + k];
    A[j * 7] = sqrt(t);
    for (int r = j + 1; r < 6; r++) { double u = A[r * 6 + j]; for (int k = 0; k < j; k++) u -= A[r * 6 + k] * A[j * 6 + k]; A[r * 6 + j] = u / A[j * 7]; }
  }
  for (int c = 0; c < 6; c++)
    for (int r = 0; r < 6; r++) {
      double t = r == c ? 1.0 : 0.0;
      for (int k = c; k < r; k++) t -= A[r * 6 + k] * Li[k * 6 + c];
      Li[r * 6 + c] = r < c ? 0.0 : t / A[r * 7];
    }
  for (int r = 0; r < 6; r++) for (int c = 0; c <= r; c++) {   // (L L^T)^-1 = L^-T L^-1
    double t = 0;
    for (int k = r; k < 6; k++) t += Li[k * 6 + r] * Li[k * 6 + c];
    cov[(size_t)e * 21 + r * (r + 1) / 2 + c] = t;
  }
}

D2BA_DEV int pcm_group_of(const long long *off, int G, long long t) {   // the g with off[g] <= t < off[g + 1]
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= t) lo = mid; else hi = mid - 1; }
  return lo;
}

// one warp per adjacency word (row i, columns 32 w .. 32 w + 31 of a group): the word is a ballot, so no atomics.  Cell (i, j)
// is the pair with edge1 = max(i, j); the smd of j < i is kept for d2pgo_debug_pcm_smd.
__global__ void __launch_bounds__(256) k_pcm_pairs(PcmDev d, int G, long long n_words) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= n_words) return;
  const int g = pcm_group_of(d.g_word, G, t);
  const int base = d.g_loop[g], L = d.g_loop[g + 1] - base, W = (L + 31) >> 5;
  const long long local = t - d.g_word[g];
  const int i = (int)(local / W), j = (int)(local % W) * 32 + lane;
  bool ok = false;
  if (j < L && j != i) {
    const double s = pcm_smd(d, base + max(i, j), base + min(i, j));
    ok = s < d.thr;
    if (j < i) d.smd[d.g_smd[g] + (long long)i * (i - 1) / 2 + j] = s;
  }
  const unsigned word = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) d.adj[t] = word;
}

__global__ void k_pcm_degree(int G, const int *g_loop, const long long *g_word, const unsigned *adj, int *deg) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g_loop[G]) return;
  int lo = 0, hi = G - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (g_loop[mid] <= e) lo = mid; else hi = mid - 1; }
  const int L = g_loop[lo + 1] - g_loop[lo], W = (L + 31) >> 5;
  const unsigned *row = adj + g_word[lo] + (long long)(e - g_loop[lo]) * W;
  int c = 0;
  for (int k = 0; k < W; k++) c += __popc(row[k]);
  deg[e] = c;
}

// FMC's greedy from seed s under the running maximum m (findCliqueHeu.cpp:146-239): C = N(s) & {deg >= m}; repeat
// v = max C, C &= N(v).  One warp; C in shared memory, word k owned by lane k % 32.  Returns the clique size 1 + picks, or 0
// once the clique can no longer exceed m (1 + picks + |C| <= m): such a seed is never taken, so stopping early changes nothing.
D2BA_DEV int pcm_greedy(int s, int m, const unsigned *rows, int W, const unsigned *degmask, unsigned *C, int lane, long long *rounds, unsigned char *member) {
  for (int k = lane; k < W; k += 32) C[k] = rows[(size_t)s * W + k] & degmask[k];
  if (member && lane == 0) member[s] = 1;
  int picks = 0;
  for (;;) {
    int cnt = 0, hi = -1;
    for (int k = lane; k < W; k += 32) { const unsigned c = C[k]; cnt += __popc(c); if (c) hi = k * 32 + 31 - __clz(c); }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if (1 + picks + cnt <= m) return 0;
    if (cnt == 0) return 1 + picks;
    if (member && lane == 0) member[hi] = 1;
    picks++; (*rounds)++;
    for (int k = lane; k < W; k += 32) C[k] &= rows[(size_t)hi * W + k];
  }
}

D2BA_DEV void pcm_degmask(unsigned *degmask, const int *deg, int L, int W, int m) {   // bit u: u < L and deg(u) >= m
  for (int k = threadIdx.x; k < W; k += blockDim.x) {
    unsigned w = 0;
    for (int b = 0; b < 32; b++) { const int u = k * 32 + b; if (u < L && deg[u] >= m) w |= 1u << b; }
    degmask[k] = w;
  }
}

// one CTA per group: FMC maxCliqueHeu, exactly.  Seeds are taken kPcmWarps at a time under the current m; the first of them
// (by index) whose clique exceeds m commits, and the seeds after it are examined again under the new m.  The committed seed's
// clique is rebuilt at the end under the m it was found with.  stats[g] = {sum of degrees, greedy rounds}.
__global__ void __launch_bounds__(kPcmWarps * 32) k_pcm_clique(const int *g_loop, const long long *g_word, const unsigned *adj, const int *deg_all, unsigned char *inlier, long long *stats) {
  extern __shared__ unsigned pcm_smem[];
  __shared__ int s_size[kPcmWarps], s_m, s_best, s_best_m, s_next;
  __shared__ long long s_part[kPcmWarps * 32];
  const int g = blockIdx.x, base = g_loop[g], L = g_loop[g + 1] - base, W = (L + 31) >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned *rows = adj + g_word[g];
  const int *deg = deg_all + base;
  unsigned *degmask = pcm_smem, *C = pcm_smem + W * (1 + warp);
  long long rounds = 0, dsum = 0;
  for (int k = threadIdx.x; k < L; k += blockDim.x) { inlier[base + k] = 0; dsum += deg[k]; }
  if (threadIdx.x == 0) { s_m = -1; s_best = -1; s_best_m = -1; }
  pcm_degmask(degmask, deg, L, W, -1);
  __syncthreads();
  for (int s0 = 0; s0 < L;) {
    const int m = s_m, s = s0 + warp;
    int size = 0;
    if (s < L && !(m > deg[s])) size = pcm_greedy(s, m, rows, W, degmask, C, lane, &rounds, nullptr);   // Pruning 1
    if (lane == 0) s_size[warp] = size;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_next = s0 + kPcmWarps;
      for (int w = 0; w < kPcmWarps; w++)
        if (s_size[w] > m) { s_best = s0 + w; s_best_m = m; s_m = s_size[w]; s_next = s0 + w + 1; break; }
    }
    __syncthreads();
    if (s_m != m) { pcm_degmask(degmask, deg, L, W, s_m); __syncthreads(); }
    s0 = s_next;
    __syncthreads();
  }
  if (s_best >= 0) {
    pcm_degmask(degmask, deg, L, W, s_best_m);
    __syncthreads();
    if (warp == 0) { long long dummy = 0; pcm_greedy(s_best, s_best_m, rows, W, degmask, C, lane, &dummy, inlier + base); }
  }
  s_part[threadIdx.x] = lane == 0 ? rounds : 0;   // every lane of a warp counted the same rounds
  __syncthreads();
  if (threadIdx.x == 0) { long long r = 0; for (int k = 0; k < kPcmWarps * 32; k++) r += s_part[k]; s_part[0] = r; }
  __syncthreads();
  const long long r = s_part[0];
  __syncthreads();
  s_part[threadIdx.x] = dsum;
  __syncthreads();
  if (threadIdx.x == 0) { long long t = 0; for (int k = 0; k < kPcmWarps * 32; k++) t += s_part[k]; stats[2 * g] = t; stats[2 * g + 1] = r; }
}

struct PcmBufs {
  Buf<int> g_loop, fa, fb, src, traj_ptr, traj, deg; Buf<long long> g_word, g_smd, stats; Buf<unsigned char> flip, inlier;
  Buf<double> rel_in, sqrt_in, rel, cov, ego, path, smd; Buf<unsigned> adj;
  long long n_smd = -1;   // tested pairs of the last d2pgo_pcm call (-1: none yet)
  cudaEvent_t ev_pair = nullptr;
  void release() {
    g_loop.release(); fa.release(); fb.release(); src.release(); traj_ptr.release(); traj.release(); deg.release(); g_word.release(); g_smd.release();
    stats.release(); flip.release(); inlier.release(); rel_in.release(); sqrt_in.release(); rel.release(); cov.release(); ego.release(); path.release();
    smd.release(); adj.release();
    if (ev_pair) cudaEventDestroy(ev_pair);
    ev_pair = nullptr;
  }
};
}  // namespace

struct d2pgo_handle {
  d2pgo_config cfg;
  int dof = 6;              // pose block size: 6 (RelPoseFactorAD on SE(3)) or 4 (RelPoseFactor4D on [x y z yaw])
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::vector<int64_t> ids; std::unordered_map<int64_t, int> index;
  std::vector<double> poses; std::vector<unsigned char> fixed;   // [N][8], the device layout of PgoDev::x
  std::vector<int> ea, eb; std::vector<double> rel, sinfo;         // rel [E][8], sinfo [E][dof^2]
  std::vector<int> gp_pose; std::vector<double> gp_u, gp_S;        // gravity priors: pose index, u_ego [G][3], S [G][9]
  Buf<double> d_gp_u, d_gp_S, d_glin[2]; Buf<int> d_gp_pose, d_prior_of;
  Buf<double> d_x[2], d_rel, d_sinfo, d_lin[2], d_g[2], d_D[2], d_Minv, d_dx, d_r, d_z, d_p, d_Ap, d_cost, d_damp, d_t, d_part, d_cost_part;
  Buf<unsigned char> d_fixed; Buf<int> d_ea, d_eb, d_inc_ptr, d_inc; Buf<PgoScalars> d_s;
  cudaGraphExec_t cg_graph[2] = {nullptr, nullptr};   // 16 CG iterations on the linearisation buffer 0 / 1 (single rank)
  double graph_tol2 = -1.0;
  bool uploaded = false;
  void *comm = nullptr; int rank = 0, nranks = 1;
  PcmBufs pcm;   // d2pgo_pcm's device buffers (independent of the poses and edges above)
};

#define PCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return 100 + (int)e_; } } while (0)

// the 6-DoF and the 4-DoF entry points each serve one kind of handle
static int pgo_want_dof(d2pgo_handle *h, int dof, const char *what) {
  if (h->dof == dof) return 0;
  h->err = std::string(what) + ": the handle was created with pose_dof = " + std::to_string(h->dof) + "; use the " +
           (h->dof == 4 ? "d2pgo_*_4d" : "6-DoF d2pgo_*") + " entry points";
  return 5;
}

static int pgo_set_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses, int width, const uint8_t *fixed, const char *what) {
  h->ids.assign(ids, ids + n); h->index.clear(); h->poses.assign((size_t)n * 8, 0.0); h->fixed.assign(n, 0);
  for (int i = 0; i < n; i++) {
    if (!h->index.emplace(ids[i], i).second) { h->err = std::string(what) + ": duplicate pose id"; return 2; }
    memcpy(&h->poses[(size_t)i * 8], poses + (size_t)i * width, (size_t)width * 8);
    h->fixed[i] = fixed ? fixed[i] : 0;
  }
  h->ea.clear(); h->eb.clear(); h->rel.clear(); h->sinfo.clear(); h->uploaded = false;
  h->gp_pose.clear(); h->gp_u.clear(); h->gp_S.clear();
  return 0;
}

static int pgo_add_edges(d2pgo_handle *h, int32_t n, const int64_t *id_a, const int64_t *id_b, const double *rel, int width, const double *sqrt_info, const char *what) {
  const int DD = h->dof * h->dof;
  for (int e = 0; e < n; e++) {
    auto a = h->index.find(id_a[e]), b = h->index.find(id_b[e]);
    if (a == h->index.end() || b == h->index.end()) { h->err = std::string(what) + ": unknown pose id"; return 2; }
    h->ea.push_back(a->second); h->eb.push_back(b->second);
    for (int k = 0; k < width; k++) h->rel.push_back(rel[(size_t)e * width + k]);
    for (int k = width; k < 8; k++) h->rel.push_back(0.0);
    for (int k = 0; k < DD; k++) h->sinfo.push_back(sqrt_info[(size_t)e * DD + k]);
  }
  h->uploaded = false;
  return 0;
}

static int pgo_get_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, double *out, int width, const char *what) {
  for (int i = 0; i < n; i++) {
    auto it = h->index.find(ids[i]);
    if (it == h->index.end()) { h->err = std::string(what) + ": unknown id"; return 2; }
    memcpy(out + (size_t)i * width, &h->poses[(size_t)it->second * 8], (size_t)width * 8);
  }
  return 0;
}

extern "C" {

int d2pgo_default_config(d2pgo_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->device = 0; c->max_iterations = 20; c->pcg_max_iterations = 200; c->pcg_tolerance = 1e-8; c->lambda0 = 1e-6; c->function_tolerance = 1e-9;
  return 0;
}

int d2pgo_create(const d2pgo_config *cfg, d2pgo_handle **out) {
  if (!cfg || !out) return 1;
  if (cfg->pose_dof != 0 && cfg->pose_dof != 6 && cfg->pose_dof != 4) {
    fprintf(stderr, "d2pgo_create: pose_dof = %d (0 or 6: 6-DoF poses, 4: [x y z yaw] poses)\n", (int)cfg->pose_dof);
    return 2;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { fprintf(stderr, "d2pgo_create: no CUDA device (there is no CPU fallback)\n"); return 3; }
  if (cfg->device < 0 || cfg->device >= ndev || cudaSetDevice(cfg->device) != cudaSuccess) return 4;
  d2pgo_handle *h = new d2pgo_handle();
  h->cfg = *cfg;
  h->dof = cfg->pose_dof == 4 ? 4 : 6;
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return 6; }
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  *out = h;
  return 0;
}

int d2pgo_destroy(d2pgo_handle *h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  cudaStreamSynchronize(h->stream);
  if (h->comm) nccl_comm_destroy(h->comm);
  for (int b = 0; b < 2; b++) { h->d_x[b].release(); h->d_g[b].release(); h->d_D[b].release(); h->d_lin[b].release(); if (h->cg_graph[b]) cudaGraphExecDestroy(h->cg_graph[b]); }
  h->d_damp.release(); h->d_t.release(); h->d_part.release(); h->d_cost_part.release(); h->d_inc_ptr.release(); h->d_inc.release();
  h->d_rel.release(); h->d_sinfo.release(); h->d_Minv.release(); h->d_dx.release(); h->d_r.release(); h->d_z.release(); h->d_p.release();
  h->d_Ap.release(); h->d_cost.release(); h->d_fixed.release(); h->d_ea.release(); h->d_eb.release(); h->d_s.release();
  h->d_gp_u.release(); h->d_gp_S.release(); h->d_glin[0].release(); h->d_glin[1].release(); h->d_gp_pose.release(); h->d_prior_of.release();
  h->pcm.release();
  cudaEventDestroy(h->ev0); cudaEventDestroy(h->ev1); cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

const char *d2pgo_last_error(const d2pgo_handle *h) { return h ? h->err.c_str() : "null handle"; }

int d2pgo_set_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses7, const uint8_t *fixed) {
  if (!h || n <= 0) return 1;
  if (int rc = pgo_want_dof(h, 6, "set_poses")) return rc;
  return pgo_set_poses(h, n, ids, poses7, 7, fixed, "set_poses");
}

int d2pgo_set_poses_4d(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses4, const uint8_t *fixed) {
  if (!h || n <= 0) return 1;
  if (int rc = pgo_want_dof(h, 4, "set_poses_4d")) return rc;
  return pgo_set_poses(h, n, ids, poses4, 4, fixed, "set_poses_4d");
}

int d2pgo_add_edges(d2pgo_handle *h, int32_t n, const int64_t *id_a, const int64_t *id_b, const double *rel7, const double *sqrt_info36) {
  if (!h) return 1;
  if (int rc = pgo_want_dof(h, 6, "add_edges")) return rc;
  return pgo_add_edges(h, n, id_a, id_b, rel7, 7, sqrt_info36, "add_edges");
}

int d2pgo_add_edges_4d(d2pgo_handle *h, int32_t n, const int64_t *id_a, const int64_t *id_b, const double *rel4, const double *sqrt_info16) {
  if (!h) return 1;
  if (int rc = pgo_want_dof(h, 4, "add_edges_4d")) return rc;
  return pgo_add_edges(h, n, id_a, id_b, rel4, 4, sqrt_info16, "add_edges_4d");
}

int d2pgo_comm_init(d2pgo_handle *h, const uint8_t unique_id[128], int32_t rank, int32_t nranks) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  if (nccl_comm_init(&h->comm, unique_id, rank, nranks, h->err)) return 3;
  h->rank = rank; h->nranks = nranks;
  return 0;
}

}  // extern "C"

static void pgo_drop_graphs(d2pgo_handle *h) {
  for (int b = 0; b < 2; b++) if (h->cg_graph[b]) { cudaGraphExecDestroy(h->cg_graph[b]); h->cg_graph[b] = nullptr; }
}

static int pgo_upload(d2pgo_handle *h) {
  const size_t N = h->ids.size(), E = h->ea.size(), nbp = (N + 127) / 128, nbe = (E + 127) / 128;
  const size_t D = h->dof, DD = D * D;
  pgo_drop_graphs(h);
  for (int b = 0; b < 2; b++) { PCK(h->d_x[b].alloc(N * 8)); PCK(h->d_g[b].alloc(N * D)); PCK(h->d_D[b].alloc(N * DD)); PCK(h->d_lin[b].alloc(E * (D + 2 * DD))); }
  PCK(h->d_rel.alloc(E * 8)); PCK(h->d_sinfo.alloc(E * DD)); PCK(h->d_Minv.alloc(N * DD));
  PCK(h->d_dx.alloc(N * D)); PCK(h->d_r.alloc(N * D)); PCK(h->d_z.alloc(N * D)); PCK(h->d_p.alloc(N * D)); PCK(h->d_Ap.alloc(N * D)); PCK(h->d_cost.alloc(2));
  const size_t G = h->gp_pose.size(), nbg = (G + 127) / 128;
  PCK(h->d_damp.alloc(N * D)); PCK(h->d_t.alloc(E * 2 * D)); PCK(h->d_part.alloc(5 * nbp)); PCK(h->d_cost_part.alloc(nbe + nbg + 1));
  PCK(h->d_fixed.alloc(N)); PCK(h->d_ea.alloc(E)); PCK(h->d_eb.alloc(E)); PCK(h->d_s.alloc(1)); PCK(h->d_inc_ptr.alloc(N + 1)); PCK(h->d_inc.alloc(2 * E));
  // incidence lists (pose -> its edges, ascending edge order): the fixed summation order of every product
  std::vector<int> ptr(N + 1, 0), inc(2 * E);
  for (size_t e = 0; e < E; e++) { ptr[h->ea[e] + 1]++; ptr[h->eb[e] + 1]++; }
  for (size_t i = 0; i < N; i++) ptr[i + 1] += ptr[i];
  { std::vector<int> fill(ptr.begin(), ptr.end() - 1);
    for (size_t e = 0; e < E; e++) { inc[fill[h->ea[e]]++] = (int)(e << 1); inc[fill[h->eb[e]]++] = (int)(e << 1 | 1); } }
  PCK(cudaMemcpyAsync(h->d_x[0].p, h->poses.data(), N * 64, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(h->d_fixed.p, h->fixed.data(), N, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(h->d_inc_ptr.p, ptr.data(), (N + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  if (E) {
    PCK(cudaMemcpyAsync(h->d_inc.p, inc.data(), 2 * E * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_ea.p, h->ea.data(), E * 4, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(h->d_eb.p, h->eb.data(), E * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_rel.p, h->rel.data(), E * 64, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(h->d_sinfo.p, h->sinfo.data(), E * DD * 8, cudaMemcpyHostToDevice, h->stream));
  }
  std::vector<int> prior_of;
  if (G) {   // gravity priors: records and the per-pose index
    PCK(h->d_gp_pose.alloc(G)); PCK(h->d_gp_u.alloc(G * 3)); PCK(h->d_gp_S.alloc(G * 9)); PCK(h->d_prior_of.alloc(N));
    for (int b = 0; b < 2; b++) PCK(h->d_glin[b].alloc(G * 12));
    prior_of.assign(N, -1);
    for (size_t k = 0; k < G; k++) prior_of[h->gp_pose[k]] = (int)k;
    PCK(cudaMemcpyAsync(h->d_gp_pose.p, h->gp_pose.data(), G * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_gp_u.p, h->gp_u.data(), G * 24, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_gp_S.p, h->gp_S.data(), G * 72, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_prior_of.p, prior_of.data(), N * 4, cudaMemcpyHostToDevice, h->stream));
  }
  PCK(cudaStreamSynchronize(h->stream));   // ptr / inc / prior_of go out of scope
  h->uploaded = true;
  return 0;
}

static PgoDev pgo_view(d2pgo_handle *h, int cur) {
  PgoDev d; memset(&d, 0, sizeof d);
  d.n_pose = (int)h->ids.size(); d.n_edge = (int)h->ea.size(); d.x = h->d_x[cur].p; d.fixed = h->d_fixed.p; d.ea = h->d_ea.p; d.eb = h->d_eb.p;
  d.rel = h->d_rel.p; d.sinfo = h->d_sinfo.p; d.lin = h->d_lin[cur].p; d.Minv = h->d_Minv.p; d.dx = h->d_dx.p; d.r = h->d_r.p; d.z = h->d_z.p; d.p = h->d_p.p;
  d.Ap = h->d_Ap.p; d.s = h->d_s.p; d.damp = h->d_damp.p; d.t = h->d_t.p; d.inc_ptr = h->d_inc_ptr.p; d.inc = h->d_inc.p;
  d.nbp = (d.n_pose + 127) / 128; d.rz_part = h->d_part.p; d.rr_part = h->d_part.p + 2 * (size_t)d.nbp; d.pAp_part = h->d_part.p + 4 * (size_t)d.nbp;
  return d;
}

static PgoPriorDev pgo_prior_view(d2pgo_handle *h, int cur) {
  PgoPriorDev pr;
  pr.n_prior = (int)h->gp_pose.size(); pr.pose = h->d_gp_pose.p; pr.prior_of = h->d_prior_of.p; pr.u = h->d_gp_u.p; pr.S = h->d_gp_S.p; pr.lin = h->d_glin[cur].p;
  return pr;
}

// cost (+ lin records, gradient, block diagonal of buffer `b`) at pose buffer `b`; all-reduced across the ranks.  GRAV: this
// rank has gravity priors (their cost partials follow the edges', their terms enter g and D after each pose's edges).
template <class P, bool GRAV>
static int pgo_linearize(d2pgo_handle *h, int b, int want_jac, double *cost) {
  constexpr int D = P::D;
  PgoDev d = pgo_view(h, b);
  const PgoPriorDev pr = pgo_prior_view(h, b);
  const size_t N = h->ids.size();
  const int nbe = (d.n_edge + 127) / 128, nbg = GRAV ? (pr.n_prior + 127) / 128 : 0;
  if (d.n_edge > 0) k_pgo_lin<P><<<nbe, 128, 0, h->stream>>>(d, h->d_cost_part.p, want_jac);
  if (nbg > 0) k_pgo_prior_lin<<<nbg, 128, 0, h->stream>>>(d, h->d_cost_part.p + nbe, want_jac, pr);
  k_pgo_sum<<<1, 128, 0, h->stream>>>(h->d_cost_part.p, nbe + nbg, h->d_cost.p);
  if (want_jac) k_pgo_gD<P, GRAV><<<d.nbp, 128, 0, h->stream>>>(d, h->d_g[b].p, h->d_D[b].p, pr);
  if (h->comm) {
    if (nccl_allreduce_f64(h->comm, h->d_cost.p, 1, h->stream)) { h->err = "ncclAllReduce(cost) failed"; return 40; }
    if (want_jac && (nccl_allreduce_f64(h->comm, h->d_g[b].p, N * D, h->stream) || nccl_allreduce_f64(h->comm, h->d_D[b].p, N * D * D, h->stream))) { h->err = "ncclAllReduce(g, D) failed"; return 40; }
  }
  PCK(cudaMemcpyAsync(cost, h->d_cost.p, 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  return 0;
}

constexpr int kCgChunk = 16;   // CG iterations between two looks at the convergence flag (one graph launch on a single rank)

template <class P, bool GRAV>
static int pgo_cg_chunk(d2pgo_handle *h, const PgoDev &d, const PgoPriorDev &pr, double tol2) {
  const int ge = (d.n_edge + 127) / 128;
  for (int k = 0; k < kCgChunk; k++) {
    const int par = k & 1;
    if (d.n_edge > 0) k_pgo_cg_edge<P><<<ge, 128, 0, h->stream>>>(d, par, tol2);
    if (h->comm) {
      k_pgo_cg_pose<P, true, GRAV><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2, pr);
      // every rank holds the same r, z, p (the all-reduced products are bitwise identical), so all of them reach the same
      // `done` decision at the same iteration and the collective below is always matched
      if (nccl_allreduce_f64(h->comm, d.Ap, (size_t)d.n_pose * P::D, h->stream)) { h->err = "ncclAllReduce(Ap) failed"; return 40; }
      k_pgo_cg_pAp<P><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2);
    } else k_pgo_cg_pose<P, false, GRAV><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2, pr);
    k_pgo_cg_step<P><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2);
  }
  return 0;
}

// the LM loop, shared by both pose parameterisations (P = PgoEdge6 / PgoEdge4) and by 6-DoF graphs with gravity priors (GRAV)
template <class P, bool GRAV>
static int pgo_solve(d2pgo_handle *h, d2pgo_report *rep) {
  int rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  const int N = (int)h->ids.size();
  const int gp = (N + 127) / 128;
  d2pgo_report R; memset(&R, 0, sizeof R);
  PCK(cudaEventRecord(h->ev0, h->stream));
  int cur = 0;                    // buffer (poses, lin records, g, D) of the accepted point
  double cost = 0, lambda = h->cfg.lambda0;
  if ((rc = pgo_linearize<P, GRAV>(h, cur, 1, &cost))) return rc;
  R.initial_cost = cost;
  const double tol2 = h->cfg.pcg_tolerance * h->cfg.pcg_tolerance;
  if (tol2 != h->graph_tol2) { pgo_drop_graphs(h); h->graph_tol2 = tol2; }
  for (int it = 0; it < h->cfg.max_iterations; it++) {
    PgoDev d = pgo_view(h, cur);
    const PgoPriorDev pr = pgo_prior_view(h, cur);
    // (J^T J + lambda diag D) dx = -g by block-Jacobi preconditioned CG; J^T J is never formed
    k_pgo_precond<P><<<gp, 128, 0, h->stream>>>(d, h->d_D[cur].p, lambda);
    k_pgo_cg_init<P><<<gp, 128, 0, h->stream>>>(d, h->d_g[cur].p);
    k_pgo_cg_init2<<<1, 128, 0, h->stream>>>(d);
    PgoScalars s; memset(&s, 0, sizeof s);
    for (int k = 0; k < h->cfg.pcg_max_iterations; k += kCgChunk) {
      if (!h->comm) {
        if (!h->cg_graph[cur]) {
          cudaGraph_t g;
          PCK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
          pgo_cg_chunk<P, GRAV>(h, d, pr, tol2);
          PCK(cudaStreamEndCapture(h->stream, &g));
          PCK(cudaGraphInstantiate(&h->cg_graph[cur], g, 0));
          cudaGraphDestroy(g);
        }
        PCK(cudaGraphLaunch(h->cg_graph[cur], h->stream));
      } else if ((rc = pgo_cg_chunk<P, GRAV>(h, d, pr, tol2))) return rc;
      PCK(cudaMemcpyAsync(&s, h->d_s.p, sizeof s, cudaMemcpyDeviceToHost, h->stream));
      PCK(cudaStreamSynchronize(h->stream));
      if (s.done) break;   // identical on every rank (see pgo_cg_chunk)
    }
    k_pgo_retract<P><<<gp, 128, 0, h->stream>>>(d, h->d_x[1 - cur].p);
    double cand = 0;
    if ((rc = pgo_linearize<P, GRAV>(h, 1 - cur, 1, &cand))) return rc;
    R.pcg_iterations += s.iters; R.iterations++;
    if (cand < cost && isfinite(cand)) {
      const double rel_dec = (cost - cand) / (cost > 0 ? cost : 1.0);
      cur = 1 - cur; cost = cand; R.accepted++;
      lambda = lambda > 0 ? fmax(lambda / 3.0, 1e-12) : 0.0;
      if (rel_dec < h->cfg.function_tolerance) { R.converged = 1; break; }
    } else {
      lambda = lambda > 0 ? lambda * 4.0 : 1e-4;
      if (lambda > 1e8) break;
    }
  }
  PCK(cudaEventRecord(h->ev1, h->stream));
  PCK(cudaMemcpyAsync(h->poses.data(), h->d_x[cur].p, (size_t)N * 64, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  if (cur != 0) PCK(cudaMemcpy(h->d_x[0].p, h->d_x[1].p, (size_t)N * 64, cudaMemcpyDeviceToDevice));   // a following solve starts from buffer 0
  float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  R.final_cost = cost; R.device_ms = ms;
  if (rep) *rep = R;
  return 0;
}

extern "C" {

int d2pgo_solve(d2pgo_handle *h, d2pgo_report *rep) {
  if (!h || h->ids.empty()) return 1;
  cudaSetDevice(h->cfg.device);
  if (h->dof == 4) return pgo_solve<PgoEdge4, false>(h, rep);
  return h->gp_pose.empty() ? pgo_solve<PgoEdge6, false>(h, rep) : pgo_solve<PgoEdge6, true>(h, rep);
}

int d2pgo_get_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, double *out) {
  if (!h) return 1;
  if (int rc = pgo_want_dof(h, 6, "get_poses")) return rc;
  return pgo_get_poses(h, n, ids, out, 7, "get_poses");
}

int d2pgo_get_poses_4d(d2pgo_handle *h, int32_t n, const int64_t *ids, double *poses4_out) {
  if (!h) return 1;
  if (int rc = pgo_want_dof(h, 4, "get_poses_4d")) return rc;
  return pgo_get_poses(h, n, ids, poses4_out, 4, "get_poses_4d");
}

int d2pgo_debug_edges(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  cudaSetDevice(h->cfg.device);
  int rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  const size_t E = h->ea.size(), W = (size_t)h->dof + 2 * (size_t)h->dof * h->dof;   // 78 (6-DoF) or 36 (4-DoF) per edge
  if ((size_t)out_doubles < E * W) { h->err = "debug_edges: buffer too small"; return 2; }
  double cost;
  if ((rc = h->dof == 4 ? pgo_linearize<PgoEdge4, false>(h, 0, 1, &cost) : pgo_linearize<PgoEdge6, false>(h, 0, 1, &cost))) return rc;
  std::vector<double> tmp(E * W);
  PCK(cudaMemcpy(tmp.data(), h->d_lin[0].p, E * W * 8, cudaMemcpyDeviceToHost));
  for (size_t e = 0; e < E; e++) for (size_t k = 0; k < W; k++) out[e * W + k] = tmp[k * E + e];   // device layout is field-major
  return 0;
}

int d2pgo_add_gravity_priors(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *ego_poses7, const double *sqrt_info9) {
  if (!h) return 1;
  if (h->dof != 6) {
    h->err = "add_gravity_priors: the handle was created with pose_dof = 4; gravity priors act on 6-DoF poses (d2pgo skips them for 4-DoF)";
    return 5;
  }
  if (n < 0 || (n > 0 && (!ids || !ego_poses7 || !sqrt_info9))) { h->err = "add_gravity_priors: negative count or null argument"; return 1; }
  // validate the whole batch before taking any of it
  std::vector<char> taken(h->ids.size(), 0);
  for (int p : h->gp_pose) taken[p] = 1;
  std::vector<int> pose(n);
  for (int k = 0; k < n; k++) {
    const std::string which = "add_gravity_priors: prior " + std::to_string(k) + " (pose id " + std::to_string(ids[k]) + ")";
    auto it = h->index.find(ids[k]);
    if (it == h->index.end()) { h->err = which + ": unknown pose id"; return 2; }
    if (taken[it->second]) { h->err = which + ": the pose already has a gravity prior"; return 2; }
    taken[it->second] = 1; pose[k] = it->second;
    bool finite = true;
    for (int j = 0; j < 7; j++) finite = finite && std::isfinite(ego_poses7[(size_t)k * 7 + j]);
    for (int j = 0; j < 9; j++) finite = finite && std::isfinite(sqrt_info9[(size_t)k * 9 + j]);
    if (!finite) { h->err = which + ": non-finite ego pose or sqrt information"; return 2; }
    const double *q = ego_poses7 + (size_t)k * 7 + 3;
    if (!(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0)) { h->err = which + ": zero ego quaternion"; return 2; }
  }
  for (int k = 0; k < n; k++) {
    // u_ego = R(q_ego)^T e3: the third row of the normalised ego attitude's rotation matrix (Swarm::Pose::R, Eigen's polynomial)
    const double *e = ego_poses7 + (size_t)k * 7 + 3;
    const double s = 1.0 / std::sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2] + e[3] * e[3]);
    const double x = e[0] * s, y = e[1] * s, z = e[2] * s, w = e[3] * s;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    h->gp_pose.push_back(pose[k]);
    h->gp_u.push_back(tz * x - ty * w); h->gp_u.push_back(tz * y + tx * w); h->gp_u.push_back(1 - (tx * x + ty * y));
    for (int j = 0; j < 9; j++) h->gp_S.push_back(sqrt_info9[(size_t)k * 9 + j]);
  }
  if (n > 0) h->uploaded = false;
  return 0;
}

int d2pgo_debug_gravity_priors(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  if (h->dof != 6) { h->err = "debug_gravity_priors: the handle was created with pose_dof = 4 (no gravity priors)"; return 5; }
  const size_t G = h->gp_pose.size();
  if ((size_t)out_doubles < G * 21) { h->err = "debug_gravity_priors: buffer too small: " + std::to_string(G * 21) + " doubles needed"; return 2; }
  if (!G) return 0;
  cudaSetDevice(h->cfg.device);
  int rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  double cost;
  if ((rc = pgo_linearize<PgoEdge6, true>(h, 0, 1, &cost))) return rc;
  std::vector<double> tmp(G * 12);
  PCK(cudaMemcpy(tmp.data(), h->d_glin[0].p, G * 12 * 8, cudaMemcpyDeviceToHost));
  for (size_t k = 0; k < G; k++) {   // device layout is field-major [12][G]: r(3), J_theta (3x3)
    double *o = out + k * 21;
    for (int a = 0; a < 3; a++) o[a] = tmp[a * G + k];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 6; b++) o[3 + a * 6 + b] = b < 3 ? 0.0 : tmp[(3 + a * 3 + b - 3) * G + k];
  }
  return 0;
}

}  // extern "C"

// ---- PCM host side
static int pcm_fail(d2pgo_handle *h, int rc, const std::string &msg) { h->err = msg; return rc; }

// FMC on groups already in h->pcm (g_loop, g_word, adj): degrees, one clique CTA per group; inlier flags by slot, stats per group
static int pcm_run_clique(d2pgo_handle *h, int G, int n, int max_w) {
  PcmBufs &P = h->pcm;
  PCK(P.deg.alloc(n)); PCK(P.inlier.alloc(n)); PCK(P.stats.alloc(2 * (size_t)G));
  if (n > 0) k_pcm_degree<<<(n + 255) / 256, 256, 0, h->stream>>>(G, P.g_loop.p, P.g_word.p, P.adj.p, P.deg.p);
  if (G > 0) k_pcm_clique<<<G, kPcmWarps * 32, (size_t)(1 + kPcmWarps) * max_w * 4, h->stream>>>(P.g_loop.p, P.g_word.p, P.adj.p, P.deg.p, P.inlier.p, P.stats.p);
  PCK(cudaGetLastError());
  return 0;
}

extern "C" {

int d2pgo_default_pcm_config(d2pgo_pcm_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->pcm_thres = 1.635; c->pos_covariance_per_meter = 4e-3; c->yaw_covariance_per_meter = 4e-5;
  return 0;
}

int d2pgo_pcm(d2pgo_handle *h, const d2pgo_pcm_config *cfg, int32_t n_frames, const int64_t *frame_ids, const int32_t *frame_agent, const double *ego_poses7,
              int32_t n_loops, const int64_t *kf_a, const int64_t *kf_b, const double *rel7, const double *sqrt_info36, uint8_t *inlier_out, d2pgo_pcm_report *rep) {
  if (!h) return 1;
  if (!cfg || n_frames < 0 || n_loops < 0 || (n_frames && (!frame_ids || !frame_agent || !ego_poses7)) ||
      (n_loops && (!kf_a || !kf_b || !rel7 || !sqrt_info36 || !inlier_out)))
    return pcm_fail(h, 1, "pcm: null argument or negative count");
  // the reference keeps pcm_thres in a float (SwarmLocalOutlierRejectionParams, d2pgo_config.h); the test is smd < that float
  const double thr = (double)(float)cfg->pcm_thres;
  if (!(std::isfinite(thr) && thr > 0.0)) return pcm_fail(h, 2, "pcm: pcm_thres must be finite and positive");
  if (!(std::isfinite(cfg->pos_covariance_per_meter) && cfg->pos_covariance_per_meter >= 0.0 && std::isfinite(cfg->yaw_covariance_per_meter) && cfg->yaw_covariance_per_meter >= 0.0))
    return pcm_fail(h, 2, "pcm: covariance rates must be finite and non-negative");
  cudaSetDevice(h->cfg.device);
  PcmBufs &P = h->pcm;
  P.n_smd = -1;
  // keyframes -> (drone, position in its trajectory = order of appearance)
  std::unordered_map<int64_t, int> fidx;
  std::unordered_map<int32_t, int> drone_of;
  std::vector<std::vector<int>> trajs;
  for (int f = 0; f < n_frames; f++) {
    if (!fidx.emplace(frame_ids[f], f).second) return pcm_fail(h, 3, "pcm: duplicate keyframe id " + std::to_string(frame_ids[f]));
    auto it = drone_of.emplace(frame_agent[f], (int)trajs.size());
    if (it.second) trajs.emplace_back();
    trajs[it.first->second].push_back(f);
  }
  // groups: unordered drone pairs, numbered by first appearance; a group's loops keep their input order
  std::unordered_map<uint64_t, int> gid;
  std::vector<int> lg(n_loops), la(n_loops), lb(n_loops), gsize;
  std::vector<uint64_t> gkey;
  for (int e = 0; e < n_loops; e++) {
    auto a = fidx.find(kf_a[e]), b = fidx.find(kf_b[e]);
    if (a == fidx.end() || b == fidx.end())
      return pcm_fail(h, 3, "pcm: loop " + std::to_string(e) + " names unknown keyframe id " + std::to_string(a == fidx.end() ? kf_a[e] : kf_b[e]));
    la[e] = a->second; lb[e] = b->second;
    const uint32_t x = (uint32_t)frame_agent[la[e]], y = (uint32_t)frame_agent[lb[e]];
    const uint64_t key = (uint64_t)std::min(x, y) << 32 | std::max(x, y);
    auto it = gid.emplace(key, (int)gsize.size());
    if (it.second) { gsize.push_back(0); gkey.push_back(key); }
    lg[e] = it.first->second; gsize[lg[e]]++;
  }
  const int G = (int)gsize.size();
  std::vector<int> g_loop(G + 1, 0); std::vector<long long> g_word(G + 1, 0), g_smd(G + 1, 0);
  int max_w = 1;
  for (int g = 0; g < G; g++) {
    const long long L = gsize[g], W = (L + 31) / 32;
    if (L > kPcmMaxGroup)
      return pcm_fail(h, 4, "pcm: the group of drones " + std::to_string((int32_t)(gkey[g] >> 32)) + " and " + std::to_string((int32_t)(gkey[g] & 0xffffffffu)) + " has " +
                                std::to_string(L) + " loops; at most " + std::to_string(kPcmMaxGroup) + " are supported");
    g_loop[g + 1] = g_loop[g] + (int)L; g_word[g + 1] = g_word[g] + L * W; g_smd[g + 1] = g_smd[g] + L * (L - 1) / 2;
    max_w = std::max(max_w, (int)W);
  }
  std::vector<int> src(n_loops), sfa(n_loops), sfb(n_loops), fill(g_loop.begin(), g_loop.end() - 1);
  std::vector<unsigned char> flip(n_loops);
  for (int e = 0; e < n_loops; e++) {
    const int s = fill[lg[e]]++;
    src[s] = e; sfa[s] = la[e]; sfb[s] = lb[e]; flip[s] = frame_agent[la[e]] > frame_agent[lb[e]];
  }
  std::vector<int> traj_ptr(1, 0), traj;
  for (auto &t : trajs) { traj.insert(traj.end(), t.begin(), t.end()); traj_ptr.push_back((int)traj.size()); }
  std::vector<double> ego((size_t)n_frames * 8, 0.0);
  for (int f = 0; f < n_frames; f++) memcpy(&ego[(size_t)f * 8], ego_poses7 + (size_t)f * 7, 56);
  const size_t n = n_loops, F = n_frames;
  PCK(P.g_loop.alloc(G + 1)); PCK(P.g_word.alloc(G + 1)); PCK(P.g_smd.alloc(G + 1)); PCK(P.fa.alloc(n)); PCK(P.fb.alloc(n)); PCK(P.src.alloc(n)); PCK(P.flip.alloc(n));
  PCK(P.rel_in.alloc(n * 7)); PCK(P.sqrt_in.alloc(n * 36)); PCK(P.rel.alloc(n * 8)); PCK(P.cov.alloc(n * 21)); PCK(P.ego.alloc(F * 8)); PCK(P.path.alloc(F));
  PCK(P.traj_ptr.alloc(traj_ptr.size())); PCK(P.traj.alloc(F)); PCK(P.adj.alloc(g_word[G])); PCK(P.smd.alloc(g_smd[G]));
  if (!P.ev_pair) PCK(cudaEventCreate(&P.ev_pair));
  PCK(cudaMemcpyAsync(P.g_loop.p, g_loop.data(), (G + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_word.p, g_word.data(), (G + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_smd.p, g_smd.data(), (G + 1) * 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.traj_ptr.p, traj_ptr.data(), traj_ptr.size() * 4, cudaMemcpyHostToDevice, h->stream));
  if (F) {
    PCK(cudaMemcpyAsync(P.traj.p, traj.data(), F * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.ego.p, ego.data(), F * 64, cudaMemcpyHostToDevice, h->stream));
  }
  if (n) {
    PCK(cudaMemcpyAsync(P.fa.p, sfa.data(), n * 4, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.fb.p, sfb.data(), n * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.src.p, src.data(), n * 4, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.flip.p, flip.data(), n, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(P.rel_in.p, rel7, n * 56, cudaMemcpyHostToDevice, h->stream)); PCK(cudaMemcpyAsync(P.sqrt_in.p, sqrt_info36, n * 288, cudaMemcpyHostToDevice, h->stream));
  }
  PcmDev d;
  d.g_loop = P.g_loop.p; d.g_word = P.g_word.p; d.g_smd = P.g_smd.p; d.fa = P.fa.p; d.fb = P.fb.p; d.flip = P.flip.p; d.rel = P.rel.p; d.cov = P.cov.p;
  d.ego = P.ego.p; d.path = P.path.p; d.adj = P.adj.p; d.deg = P.deg.p; d.smd = P.smd.p;
  d.is4 = h->dof == 4; d.thr = thr; d.pos_cov = cfg->pos_covariance_per_meter; d.yaw_cov = cfg->yaw_covariance_per_meter;
  PCK(cudaEventRecord(h->ev0, h->stream));
  if (!trajs.empty()) k_pcm_path<<<((int)trajs.size() * 32 + 255) / 256, 256, 0, h->stream>>>((int)trajs.size(), P.traj_ptr.p, P.traj.p, P.ego.p, P.path.p);
  if (n) {
    k_pcm_loop<<<((int)n + 127) / 128, 128, 0, h->stream>>>((int)n, P.src.p, P.rel_in.p, P.sqrt_in.p, P.rel.p, P.cov.p);
    const long long words = g_word[G];
    k_pcm_pairs<<<(unsigned)((words * 32 + 255) / 256), 256, 0, h->stream>>>(d, G, words);
  }
  PCK(cudaGetLastError());
  PCK(cudaEventRecord(P.ev_pair, h->stream));
  if (int rc = pcm_run_clique(h, G, (int)n, max_w)) return rc;
  PCK(cudaEventRecord(h->ev1, h->stream));
  std::vector<unsigned char> inl(n);
  std::vector<long long> stats(2 * (size_t)G);
  if (n) PCK(cudaMemcpyAsync(inl.data(), P.inlier.p, n, cudaMemcpyDeviceToHost, h->stream));
  if (G) PCK(cudaMemcpyAsync(stats.data(), P.stats.p, 16 * (size_t)G, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  d2pgo_pcm_report R; memset(&R, 0, sizeof R);
  for (size_t s = 0; s < n; s++) { inlier_out[src[s]] = inl[s]; R.inliers += inl[s]; }
  for (int g = 0; g < G; g++) { R.consistent_pairs += stats[2 * g] / 2; R.clique_rounds += stats[2 * g + 1]; }
  R.groups = G; R.pairs_tested = g_smd[G];
  float ms = 0, mp = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1); cudaEventElapsedTime(&mp, h->ev0, P.ev_pair);
  R.device_ms = ms; R.pair_ms = mp; R.clique_ms = ms - mp;
  P.n_smd = g_smd[G];
  if (rep) *rep = R;
  return 0;
}

int d2pgo_debug_pcm_smd(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  PcmBufs &P = h->pcm;
  if (P.n_smd < 0) return pcm_fail(h, 2, "debug_pcm_smd: no successful d2pgo_pcm call on this handle");
  if (out_doubles < P.n_smd) return pcm_fail(h, 2, "debug_pcm_smd: buffer too small: " + std::to_string(P.n_smd) + " doubles needed");
  cudaSetDevice(h->cfg.device);
  if (P.n_smd) PCK(cudaMemcpy(out, P.smd.p, (size_t)P.n_smd * 8, cudaMemcpyDeviceToHost));
  return 0;
}

int d2pgo_debug_pcm_clique(d2pgo_handle *h, int32_t n, const uint32_t *adj, uint8_t *member_out, int32_t *size_out) {
  if (!h) return 1;
  if (n < 0 || (n && (!adj || !member_out))) return pcm_fail(h, 1, "debug_pcm_clique: null argument or negative count");
  if (n > kPcmMaxGroup) return pcm_fail(h, 4, "debug_pcm_clique: at most " + std::to_string(kPcmMaxGroup) + " vertices are supported");
  cudaSetDevice(h->cfg.device);
  PcmBufs &P = h->pcm;
  const long long W = (n + 31) / 32;
  const int g_loop[2] = {0, n}; const long long g_word[2] = {0, n * W};
  P.n_smd = -1;   // the buffers below are shared with d2pgo_pcm
  PCK(P.g_loop.alloc(2)); PCK(P.g_word.alloc(2)); PCK(P.adj.alloc(n * W));
  PCK(cudaMemcpyAsync(P.g_loop.p, g_loop, 8, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(P.g_word.p, g_word, 16, cudaMemcpyHostToDevice, h->stream));
  if (n) PCK(cudaMemcpyAsync(P.adj.p, adj, (size_t)(n * W) * 4, cudaMemcpyHostToDevice, h->stream));
  if (int rc = pcm_run_clique(h, n ? 1 : 0, n, (int)std::max(W, 1LL))) return rc;
  if (n) PCK(cudaMemcpyAsync(member_out, P.inlier.p, n, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  int c = 0;
  for (int k = 0; k < n; k++) c += member_out[k];
  if (size_out) *size_out = c;
  return 0;
}

}  // extern "C"
