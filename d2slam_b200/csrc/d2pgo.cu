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
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <type_traits>

#include "d2ba_math.cuh"
#include "d2pgo_handle.cuh"
#include "d2pgo_chart.cuh"
#include "d2pgo_lm.cuh"

namespace d2ba {
// NCCL through the dlopen'ed entry points of d2ba_host.cu
int nccl_comm_init(void **comm, const uint8_t *unique_id, int rank, int nranks, std::string &err);
int nccl_allreduce_f64(void *comm, double *buf, size_t n, cudaStream_t s);
void nccl_comm_destroy(void *comm);
}  // namespace d2ba
using namespace d2ba;
using namespace d2pgo_host;

namespace {

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

// ---- ARock (d2pgo's pgo_mode 1, ARockSolver / ARockPGO): proximal terms of one agent's local problem and its dual update.
// A dual (neighbour, frame) holds y_l (sent to the neighbour) and y_r (received); its proximal term pulls the frame's pose, in
// dual coordinates, towards y_r.  Dual coordinates: 4-DoF the pose [x y z yaw] itself (POSE_4D); 6-DoF [p ; theta] with
// R = R(q_init) Exp(theta) (POSE_PERTURB_6D, pgostate.hpp:35-46).  The proximal terms run in kernels of their own after the
// edge / prior kernels (k_pgo_arock_gD after k_pgo_gD, k_pgo_arock_cg_pAp in place of the damping pass), so the kernels of a
// graph without ARock are untouched.
struct PgoArockDev {
  int n_dual;
  const int *pose;            // [K] pose index of each dual
  const int *ptr, *of;        // CSR pose -> its duals, ascending dual index
  const double *yr;           // [K][D] remote duals: the proximal targets
  double *yl;                 // [K][D] local duals
  const double *qinit;        // [N][4] attitude the 6-DoF perturbation is taken from (unit, xyzw)
  double *lin;                // [D + D^2][K] field-major: r(D), J (DxD row-major)
  double wT, wR;              // residual weights: 4-DoF rho_T, rho_theta (ConsenusPoseFactor4D); 6-DoF sqrt of them (NormalPrior A)
  double eta;
};

// theta = Log(q_init^-1 q) (principal, |theta| <= pi) and, with Jinv, J_r^-1(theta) = d theta / d dtheta of the right
// perturbation q (x) Exp(dtheta): I + [theta]x / 2 + c2 [theta]x^2, c2 = 1/a^2 - (1 + cos a) / (2 a sin a), a = |theta|;
// with the half-angle quaternion (|v|, w) = (sin a/2, cos a/2) of q_init^-1 q: c2 = 1/a^2 - w / (2 a |v|) (series below 1e-2)
D2BA_DEV void arock_theta(const double *x, const double *qi, double *th, double *Jinv) {   // x: [x y z qx qy qz qw]
  Q4 e = qmul(Q4{-qi[0], -qi[1], -qi[2], qi[3]}, qload(x + 3));
  if (e.w < 0.0) e = Q4{-e.x, -e.y, -e.z, -e.w};
  const double n = sqrt(e.x * e.x + e.y * e.y + e.z * e.z);
  const double a = 2.0 * atan2(n, e.w), k = n > 0.0 ? a / n : 2.0 / e.w;
  th[0] = k * e.x; th[1] = k * e.y; th[2] = k * e.z;
  if (!Jinv) return;
  const double a2 = a * a;
  const double c2 = a < 1e-2 ? 1.0 / 12.0 + a2 / 720.0 + a2 * a2 / 30240.0 : 1.0 / a2 - e.w / (2.0 * a * n);
  const double K[9] = {0.0, -th[2], th[1], th[2], 0.0, -th[0], -th[1], th[0], 0.0};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    double k2 = 0.0;
    for (int m = 0; m < 3; m++) k2 += K[i * 3 + m] * K[m * 3 + j];
    Jinv[i * 3 + j] = (i == j ? 1.0 : 0.0) + 0.5 * K[i * 3 + j] + c2 * k2;
  }
}

// pose x in dual coordinates (D = 4: the 4-vector; D = 6: [p ; theta])
template <int D>
D2BA_DEV void arock_coord(const double *x, const double *qi, double *c) {
  for (int k = 0; k < 3; k++) c[k] = x[k];
  if constexpr (D == 4) c[3] = x[3];
  else arock_theta(x, qi, c + 3, nullptr);
}

// one proximal term at pose x, target y:
//   4-DoF ConsenusPoseFactor4D(y, rho_T, rho_theta, norm_yaw) (consenus_factor_4d.h, utils.hpp:267-280):
//     r = diag(rho_T I3, rho_theta) [y_p - p ; N(N(y_yaw) - yaw)],  J = -diag(rho_T I3, rho_theta)
//   6-DoF NormalPrior(A, y), A = diag(sqrt(rho_T) I3, sqrt(rho_theta) I3) (ARock.cpp:284-291):
//     r = A ([p ; theta] - y),  J = A blockdiag(I3, J_r^-1(theta))
template <int D>
D2BA_DEV void arock_eval(const double *x, const double *qi, const double *y, double wT, double wR, double *r, double *J) {
  for (int k = 0; k < D * D; k++) J[k] = 0.0;
  if constexpr (D == 4) {
    for (int k = 0; k < 3; k++) { r[k] = wT * (y[k] - x[k]); J[k * 5] = -wT; }
    r[3] = wR * pgo_normalize_angle(pgo_normalize_angle(y[3]) - x[3]);
    J[15] = -wR;
  } else {
    double th[3], Ji[9];
    arock_theta(x, qi, th, Ji);
    for (int k = 0; k < 3; k++) { r[k] = wT * (x[k] - y[k]); r[3 + k] = wR * (th[k] - y[3 + k]); J[k * 7] = wT; }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[(3 + i) * 6 + 3 + j] = wR * Ji[i * 3 + j];
  }
}

// linearise every proximal term at d.x: records [r | J]; cost partials go after the edges' and the priors' (k_pgo_sum)
template <int D>
__global__ void __launch_bounds__(128) k_pgo_arock_lin(PgoDev d, double *cost_part, PgoArockDev a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (k < a.n_dual) {
    const int i = a.pose[k];
    double r[D], J[D * D];
    arock_eval<D>(d.x + (size_t)i * 8, a.qinit + (size_t)i * 4, a.yr + (size_t)k * D, a.wT, a.wR, r, J);
    for (int q = 0; q < D; q++) c += 0.5 * r[q] * r[q];
    double *o = a.lin + k;
    const size_t K = (size_t)a.n_dual;
    for (int q = 0; q < D; q++) o[q * K] = r[q];
    for (int q = 0; q < D * D; q++) o[(D + q) * K] = J[q];
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}

// after k_pgo_gD: g_i += sum J^T r, D_i += sum J^T J over pose i's duals, in dual order (free poses only)
template <int D>
__global__ void __launch_bounds__(128) k_pgo_arock_gD(PgoDev d, double *g, double *Dg, PgoArockDev a) {
  constexpr int DD = D * D;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n_pose || d.fixed[i] || a.ptr[i] == a.ptr[i + 1]) return;
  double gi[D], Di[DD];
  for (int k = 0; k < D; k++) gi[k] = g[(size_t)i * D + k];
  for (int k = 0; k < DD; k++) Di[k] = Dg[(size_t)i * DD + k];
  const size_t K = (size_t)a.n_dual;
  for (int q = a.ptr[i]; q < a.ptr[i + 1]; q++) {
    const double *o = a.lin + a.of[q];
    for (int k = 0; k < D; k++) {
      const double rk = o[k * K];
      double row[D];
      for (int b = 0; b < D; b++) { row[b] = o[(D + k * D + b) * K]; gi[b] += row[b] * rk; }
      for (int b = 0; b < D; b++) for (int c = 0; c < D; c++) Di[b * D + c] += row[b] * row[c];
    }
  }
  for (int k = 0; k < D; k++) g[(size_t)i * D + k] = gi[k];
  for (int k = 0; k < DD; k++) Dg[(size_t)i * DD + k] = Di[k];
}

// after k_pgo_cg_pose<P, LOCAL = true>: Ap_i += sum J^T (J p_i) over pose i's duals, then the damping and the partials of
// p.Ap (what k_pgo_cg_pAp does for a multi-rank graph)
template <class P>
__global__ void __launch_bounds__(128) k_pgo_arock_cg_pAp(PgoDev d, int par, double tol2, PgoArockDev a) {
  constexpr int D = P::D;
  __shared__ double red[40];
  const CgView v = cg_view(d, par, tol2, red);
  if (v.done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (i < d.n_pose) {
    double p[D], y[D];
    for (int k = 0; k < D; k++) { p[k] = d.p[(size_t)i * D + k]; y[k] = d.Ap[(size_t)i * D + k]; }
    if (!d.fixed[i]) {
      const size_t K = (size_t)a.n_dual;
      for (int q = a.ptr[i]; q < a.ptr[i + 1]; q++) {
        const double *J = a.lin + (size_t)D * K + a.of[q];
        for (int k = 0; k < D; k++) {
          double j[D], t = 0.0;
          for (int b = 0; b < D; b++) { j[b] = J[(size_t)(k * D + b) * K]; t += j[b] * p[b]; }
          for (int b = 0; b < D; b++) y[b] += j[b] * t;
        }
      }
    }
    for (int k = 0; k < D; k++) {
      y[k] += d.damp[(size_t)i * D + k] * p[k];
      s += p[k] * y[k];
      d.Ap[(size_t)i * D + k] = y[k];
    }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) d.pAp_part[blockIdx.x] = s;
}

// updateDualStates (ARock.cpp:50-81) per dual at the solved poses x: y_l -= eta ((y_l + y_r) / 2 - x), x in dual coordinates,
// the operations in the reference's order and rounding (no contraction); 4-DoF: y_l's yaw normalised only once outside +-pi
template <int D>
__global__ void k_pgo_arock_update(const double *x, PgoArockDev a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.n_dual) return;
  const int i = a.pose[k];
  double c[D];
  arock_coord<D>(x + (size_t)i * 8, a.qinit + (size_t)i * 4, c);
  double *yl = a.yl + (size_t)k * D;
  const double *yr = a.yr + (size_t)k * D;
  for (int q = 0; q < D; q++) {
    const double avg = __ddiv_rn(__dadd_rn(yl[q], yr[q]), 2.0);
    yl[q] = __dsub_rn(yl[q], __dmul_rn(__dsub_rn(avg, c[q]), a.eta));
  }
  if constexpr (D == 4) if (yl[3] > M_PI || yl[3] < -M_PI) yl[3] = pgo_normalize_angle(yl[3]);
}

// every pose in dual coordinates, [N][D] (the value a dual created by scanning starts from)
template <int D>
__global__ void k_pgo_arock_coord(int n, const double *x, const double *qinit, double *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double c[D];
  arock_coord<D>(x + (size_t)i * 8, qinit + (size_t)i * 4, c);
  for (int k = 0; k < D; k++) out[(size_t)i * D + k] = c[k];
}

// ---- chordal rotation initialisation (d2pgo_rot_init; RotationInitialization<double>, rotation_initialization_base.hpp).
// One row system k at a time through the solver above: the "pose" is row k of R_f (x[0..2] of the 8 doubles), an edge's
// residual S (R_ab^T x_a - x_b) with R_ab the edge's (normalised) quaternion and S = s I3, fixed frames hold their rows as
// constants.  The residual is linear, so one Gauss-Newton step from x = 0 with CG run to a tight tolerance solves the system.
D2BA_DEV void rotinit_edge_eval(const double *xa, const double *xb, const double *rel, const double *S, double *r, double *J0, double *J1) {
  double R[9];
  q2R(qload(rel + 3), R);
  const double v[3] = {R[0] * xa[0] + R[3] * xa[1] + R[6] * xa[2] - xb[0],   // R_ab^T x_a - x_b
                       R[1] * xa[0] + R[4] * xa[1] + R[7] * xa[2] - xb[1],
                       R[2] * xa[0] + R[5] * xa[1] + R[8] * xa[2] - xb[2]};
  for (int i = 0; i < 3; i++) r[i] = S[i * 3] * v[0] + S[i * 3 + 1] * v[1] + S[i * 3 + 2] * v[2];
  if (!J0) return;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    J0[i * 3 + j] = S[i * 3] * R[j * 3] + S[i * 3 + 1] * R[j * 3 + 1] + S[i * 3 + 2] * R[j * 3 + 2];   // S R_ab^T
    J1[i * 3 + j] = -S[i * 3 + j];
  }
}
struct PgoRotRow {   // one row of R per frame, x + dx
  static constexpr int D = 3, NX = 3;
  D2BA_DEV static void eval(const double *p0, const double *p1, const double *rel, const double *S, double *r, double *J0, double *J1) { rotinit_edge_eval(p0, p1, rel, S, r, J0, J1); }
  D2BA_DEV static void plus(const double *x, const double *dx, double *o) { for (int k = 0; k < 3; k++) o[k] = x[k] + dx[k]; }
};

template <int P, int Q>
D2BA_DEV void rotinit_order(double *sv, double *A, double *V) {   // columns P < Q of A and V swapped if sv[P] < sv[Q]
  if (!(sv[P] < sv[Q])) return;
  double t = sv[P]; sv[P] = sv[Q]; sv[Q] = t;
  for (int i = 0; i < 3; i++) {
    t = A[i * 3 + P]; A[i * 3 + P] = A[i * 3 + Q]; A[i * 3 + Q] = t;
    t = V[i * 3 + P]; V[i * 3 + P] = V[i * 3 + Q]; V[i * 3 + Q] = t;
  }
}

// Utility::recoverRotationSVD (d2common/include/d2common/utils.hpp:121-129): R = U diag(1, 1, det(U V^T)) V^T of M = U S V^T,
// singular values descending (JacobiSVD's order).  One-sided (Hestenes) Jacobi on the columns of M; row-major in and out.
D2BA_DEV void rotinit_project_svd(const double *M, double *R) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int k = 0; k < 9; k++) A[k] = M[k];
  for (int sweep = 0; sweep < 16; sweep++) {
    bool rotated = false;
    for (int pq = 0; pq < 3; pq++) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double al = 0, be = 0, ga = 0;
      for (int i = 0; i < 3; i++) { al += A[i * 3 + p] * A[i * 3 + p]; be += A[i * 3 + q] * A[i * 3 + q]; ga += A[i * 3 + p] * A[i * 3 + q]; }
      if (!(fabs(ga) > 2.220446049250313e-16 * sqrt(al * be))) continue;
      rotated = true;
      const double zeta = (be - al) / (2.0 * ga);
      const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
      for (int i = 0; i < 3; i++) {
        const double ap = A[i * 3 + p], aq = A[i * 3 + q], vp = V[i * 3 + p], vq = V[i * 3 + q];
        A[i * 3 + p] = c * ap - s * aq; A[i * 3 + q] = s * ap + c * aq;
        V[i * 3 + p] = c * vp - s * vq; V[i * 3 + q] = s * vp + c * vq;
      }
    }
    if (!rotated) break;
  }
  // columns in descending singular-value order (compare-and-swap of whole columns: static indices, no local memory)
  double sv[3];
  for (int j = 0; j < 3; j++) sv[j] = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
  rotinit_order<0, 1>(sv, A, V); rotinit_order<1, 2>(sv, A, V); rotinit_order<0, 1>(sv, A, V);
  double U[9], W[9];
  for (int j = 0; j < 3; j++) {
    const double inv = sv[j] > 0.0 ? 1.0 / sv[j] : 0.0;
    for (int i = 0; i < 3; i++) { U[i * 3 + j] = A[i * 3 + j] * inv; W[i * 3 + j] = V[i * 3 + j]; }
  }
  if (!(sv[2] > 0.0)) {   // rank-deficient M: complete U by the cross product of its first two columns
    U[2] = U[3] * U[7] - U[6] * U[4]; U[5] = U[6] * U[1] - U[0] * U[7]; U[8] = U[0] * U[4] - U[3] * U[1];
  }
  const double detU = U[0] * (U[4] * U[8] - U[5] * U[7]) - U[1] * (U[3] * U[8] - U[5] * U[6]) + U[2] * (U[3] * U[7] - U[4] * U[6]);
  const double detW = W[0] * (W[4] * W[8] - W[5] * W[7]) - W[1] * (W[3] * W[8] - W[5] * W[6]) + W[2] * (W[3] * W[7] - W[4] * W[6]);
  const double d = detU * detW < 0.0 ? -1.0 : 1.0;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
    R[i * 3 + j] = U[i * 3] * W[j * 3] + U[i * 3 + 1] * W[j * 3 + 1] + d * U[i * 3 + 2] * W[j * 3 + 2];
}

// Eigen's Quaternion(const Matrix3 &) (quaternionbase_assign_impl): the trace branch, else the largest diagonal's
template <int I>
D2BA_DEV Q4 rotinit_quat_diag(const double *R) {   // the branch of the largest diagonal entry I
  constexpr int J = (I + 1) % 3, K = (J + 1) % 3;
  double q[4];   // x y z w
  double t = sqrt(R[I * 4] - R[J * 4] - R[K * 4] + 1.0);
  q[I] = 0.5 * t; t = 0.5 / t;
  q[3] = (R[K * 3 + J] - R[J * 3 + K]) * t; q[J] = (R[J * 3 + I] + R[I * 3 + J]) * t; q[K] = (R[K * 3 + I] + R[I * 3 + K]) * t;
  return Q4{q[0], q[1], q[2], q[3]};
}
D2BA_DEV Q4 rotinit_quat(const double *R) {
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0.0) {
    double t = sqrt(tr + 1.0);
    const double w = 0.5 * t;
    t = 0.5 / t;
    return Q4{(R[7] - R[5]) * t, (R[2] - R[6]) * t, (R[3] - R[1]) * t, w};
  }
  if (R[8] > (R[4] > R[0] ? R[4] : R[0])) return rotinit_quat_diag<2>(R);
  return R[4] > R[0] ? rotinit_quat_diag<1>(R) : rotinit_quat_diag<0>(R);
}

// recoverRotationLLT (rotation_initialization_base.hpp:360-389) per solved frame: M = [row 0 ; row 1 ; row 2] from the three
// row systems' solutions m0..m2 ([N][8], row at +0), its state change |R_before - M|_F / |R_before|_F (R_before: the rotation
// of the frame's normalised attitude, PGOState's rot state) into per-block partials, and the attitude x[3..6] = quaternion of
// the projected R.  The position x[0..2] is not written.
__global__ void __launch_bounds__(128) k_rotinit_project(int n, const int *frame, const double *m0, const double *m1, const double *m2, double *x, double *chg_part) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double chg = 0.0;
  if (j < n) {
    const size_t i = (size_t)frame[j];
    double M[9], R0[9], R[9];
    for (int c = 0; c < 3; c++) { M[c] = m0[i * 8 + c]; M[3 + c] = m1[i * 8 + c]; M[6 + c] = m2[i * 8 + c]; }
    Q4 q = qload(x + i * 8 + 3);
    const double qn = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    q = Q4{q.x / qn, q.y / qn, q.z / qn, q.w / qn};
    q2R(q, R0);
    double dd = 0.0, nn = 0.0;
    for (int c = 0; c < 9; c++) { dd += (R0[c] - M[c]) * (R0[c] - M[c]); nn += R0[c] * R0[c]; }
    chg = sqrt(dd) / sqrt(nn);
    rotinit_project_svd(M, R);
    const Q4 o = rotinit_quat(R);
    x[i * 8 + 3] = o.x; x[i * 8 + 4] = o.y; x[i * 8 + 5] = o.z; x[i * 8 + 6] = o.w;
  }
  chg = block_sum(chg, red);
  if (threadIdx.x == 0) chg_part[blockIdx.x] = chg;
}

// ---- distributed rotation initialisation (d2pgo_arock_rot_init_step; RotationInitARock<double>,
// rotation_initialization_arock.hpp).  A dual prior w (r_f^k - (row k of Y_r)^T) = 0 is an edge from a fixed virtual node
// (R_ab = I, S = w I3) whose value is row k of the dual's y_r; this kernel writes those values for row system k into the virtual
// nodes x[j] of the dual priors j, dual[j] being the dual of prior j in table order.
__global__ void k_rotinit_arock_targets(int n, int k, const int *dual, const double *yr, double *x) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  for (int c = 0; c < 3; c++) x[(size_t)j * 8 + c] = yr[(size_t)dual[j] * 9 + 3 * k + c];
}

// recoverRotationLLT (rotation_initialization_base.hpp:360-389) with is_multi set, per solved frame j: M from the three row
// solutions, |R_state - M|_F / |R_state|_F into per-block partials, R_state = M unprojected (the value the dual update reads),
// and, for frames this agent owns only, the attitude x[3..6] = quaternion of the projection of M.  Eigen's JacobiSVD of M = 0
// gives U = V = I, so the zero matrix projects to I (a non-main agent's first step without gravity rows has b = 0, M = 0).
__global__ void __launch_bounds__(128) k_rotinit_arock_project(int n, const int *frame, const unsigned char *owned, const double *m0,
                                                               const double *m1, const double *m2, double *rstate, double *x, double *chg_part) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double chg = 0.0;
  if (j < n) {
    const size_t i = (size_t)frame[j];
    double M[9], R[9];
    for (int c = 0; c < 3; c++) { M[c] = m0[i * 8 + c]; M[3 + c] = m1[i * 8 + c]; M[6 + c] = m2[i * 8 + c]; }
    double dd = 0.0, nn = 0.0;
    bool zero = true;
    for (int c = 0; c < 9; c++) {
      const double s = rstate[i * 9 + c];
      dd += (s - M[c]) * (s - M[c]); nn += s * s;
      rstate[i * 9 + c] = M[c];
      zero = zero && M[c] == 0.0;
    }
    chg = sqrt(dd) / sqrt(nn);
    if (owned[j]) {
      if (zero) for (int c = 0; c < 9; c++) R[c] = c % 4 == 0 ? 1.0 : 0.0;
      else rotinit_project_svd(M, R);
      const Q4 o = rotinit_quat(R);
      x[i * 8 + 3] = o.x; x[i * 8 + 4] = o.y; x[i * 8 + 5] = o.z; x[i * 8 + 6] = o.w;
    }
  }
  chg = block_sum(chg, red);
  if (threadIdx.x == 0) chg_part[blockIdx.x] = chg;
}

// updateDualStates, vector branch (ARock.cpp:63-81), per dual k on frame pose[k]: y_l -= eta ((y_l + y_r) / 2 - x) with x the
// frame's R_state (for a fixed frame, the rotation of its attitude when it entered), in the reference's order and rounding
__global__ void k_rotinit_arock_update(int n, const int *pose, const double *rstate, const double *yr, double *yl, double eta) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const double *x = rstate + (size_t)pose[k] * 9;
  for (int q = 0; q < 9; q++) {
    const double l = yl[(size_t)k * 9 + q];
    const double avg = __ddiv_rn(__dadd_rn(l, yr[(size_t)k * 9 + q]), 2.0);
    yl[(size_t)k * 9 + q] = __dsub_rn(l, __dmul_rn(__dsub_rn(avg, x[q]), eta));
  }
}

// ---- the host policy of each pose parameterisation, picked once per call by with_policy: Kern, the kernel policy of the kernels
// that read only D; the kernels that linearise, retract and update the ARock duals; the dual coordinates; the ceres minimiser's
// norms; whether the ARock q_init table holds h->qinit.  The retraction of 6-DoF (K = PgoEdge6) or 4-DoF poses: this file's kernels
template <class K> struct PgoRetraction {
  using Kern = K;
  static constexpr int D = K::D;
  static constexpr bool arock_qinit = D == 6;   // the 6-DoF dual coordinates [p ; theta] are taken from q_init
  static constexpr auto xnorm = d2pgo_lm::xnorm;
  static void lin_edges(const d2pgo_handle *, cudaStream_t st, const PgoDev &d, double *part, int want_jac) { k_pgo_lin<K><<<(d.n_edge + 127) / 128, 128, 0, st>>>(d, part, want_jac); }
  static void lin_priors(const d2pgo_handle *, cudaStream_t st, const PgoDev &d, const PgoPriorDev &pr, double *part, int want_jac) {
    k_pgo_prior_lin<<<(pr.n_prior + 127) / 128, 128, 0, st>>>(d, part, want_jac, pr);
  }
  static void lin_arock(cudaStream_t st, const PgoDev &d, const PgoArockDev &ak, double *part) { k_pgo_arock_lin<D><<<(ak.n_dual + 127) / 128, 128, 0, st>>>(d, part, ak); }
  static void retract(cudaStream_t st, const PgoDev &d, double *x_out) { k_pgo_retract<K><<<d.nbp, 128, 0, st>>>(d, x_out); }
  static void arock_update(cudaStream_t st, const double *x, const PgoArockDev &ak) { k_pgo_arock_update<D><<<(ak.n_dual + 127) / 128, 128, 0, st>>>(x, ak); }
  static int arock_coords(d2pgo_handle *h, std::vector<double> &out) {
    const size_t N = h->ids.size();
    PCK(h->d_ak_coord.alloc(N * D));
    k_pgo_arock_coord<D><<<(int)((N + 127) / 128), 128, 0, h->stream>>>((int)N, h->d_x[0].p, h->d_ak_qinit.p, h->d_ak_coord.p);
    PCK(cudaGetLastError());
    out.resize(N * D);
    PCK(cudaMemcpyAsync(out.data(), h->d_ak_coord.p, N * D * 8, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
    return 0;
  }
};

// the perturbation chart (d2pgo_set_chart), records [p, theta, 0, 0] with q_init h->d_qinit: the kernels of d2pgo_chart.cu
struct PgoChart6 {
  using Kern = PgoEdge6;
  static constexpr int D = 6;
  static constexpr bool arock_qinit = true;   // as on every 6-DoF handle, though no chart kernel reads it
  static constexpr auto xnorm = d2pgo_lm::xnorm_chart;
  static void lin_edges(const d2pgo_handle *h, cudaStream_t st, const PgoDev &d, double *part, int want_jac) {
    d2pgo_chart::edges(st, d.n_edge, d.ea, d.eb, d.x, h->d_qinit.p, d.rel, d.sinfo, d.lin, part, want_jac);
  }
  static void lin_priors(const d2pgo_handle *h, cudaStream_t st, const PgoDev &d, const PgoPriorDev &pr, double *part, int want_jac) {
    d2pgo_chart::priors(st, pr.n_prior, pr.pose, pr.u, pr.S, d.x, h->d_qinit.p, pr.lin, part, want_jac);
  }
  static void lin_arock(cudaStream_t st, const PgoDev &d, const PgoArockDev &ak, double *part) { d2pgo_chart::arock_lin(st, ak.n_dual, ak.pose, d.x, ak.yr, ak.wT, ak.wR, ak.lin, part); }
  static void retract(cudaStream_t st, const PgoDev &d, double *x_out) { d2pgo_chart::retract(st, d.n_pose, d.x, d.fixed, d.dx, x_out); }
  static void arock_update(cudaStream_t st, const double *x, const PgoArockDev &ak) { d2pgo_chart::arock_update(st, ak.n_dual, ak.pose, x, ak.yr, ak.yl, ak.eta); }
  static int arock_coords(d2pgo_handle *h, std::vector<double> &out) {   // the dual coordinates are the state [p, theta] itself
    const size_t N = h->ids.size();
    std::vector<double> x(N * 8);
    PCK(cudaMemcpyAsync(x.data(), h->d_x[0].p, N * 64, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
    out.resize(N * 6);
    for (size_t i = 0; i < N; i++) memcpy(&out[i * 6], &x[i * 8], 48);
    return 0;
  }
};

template <class K> constexpr bool kPriorKern = K::D == 6;   // k_pgo_gD and k_pgo_cg_pose have gravity-prior instantiations

}  // namespace

// the 6-DoF and the 4-DoF entry points each serve one kind of handle
static int pgo_want_dof(d2pgo_handle *h, int dof, const char *what) {
  if (h->dof == dof) return 0;
  h->err = std::string(what) + ": the handle was created with pose_dof = " + std::to_string(h->dof) + "; use the " +
           (h->dof == 4 ? "d2pgo_*_4d" : "6-DoF d2pgo_*") + " entry points";
  return 5;
}

// an ARock dual table without the duals of frames the handle no longer has
template <class Duals> static void arock_keep_present(const d2pgo_handle *h, Duals &duals) {
  for (auto it = duals.begin(); it != duals.end();) it = h->index.count(it->first.second) ? std::next(it) : duals.erase(it);
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
  arock_keep_present(h, h->pose_table.duals);   // ARock duals live on for the frames still present
  arock_keep_present(h, h->rot_table.duals);    // and so do the rotation-initialisation duals and states
  for (auto it = h->rot_state.begin(); it != h->rot_state.end();)
    it = h->index.count(it->first) ? std::next(it) : h->rot_state.erase(it);
  h->ak_n = -1;
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

// ---- the perturbation chart, host side (d2pgo_set_chart)
static bool all_finite(const double *v, size_t n) {
  for (size_t k = 0; k < n; k++) if (!std::isfinite(v[k])) return false;
  return true;
}

// a q_init as the chart keeps it: finite, non-zero, normalised (false otherwise)
static bool chart_unit(const double *q, double *out) {
  const double s2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (!all_finite(q, 4) || !(s2 > 0.0)) return false;
  const double s = 1.0 / std::sqrt(s2);
  for (int k = 0; k < 4; k++) out[k] = q[k] * s;
  return true;
}

// normalise(q_init (x) quatfromRotationVector(theta)) of a chart record [p, theta, 0, 0] (postPerturbSolve, d2pgo.cpp:616-628;
// the normalisation is Swarm::Pose's, ASSUMED)
static void chart_attitude(const double *x, const double *qi, double *q) {
  const double *th = x + 3;
  const double n = std::sqrt(th[0] * th[0] + th[1] * th[1] + th[2] * th[2]);
  double d[4];   // x y z w
  if (n < 1e-2) { d[0] = th[0] / 2.0; d[1] = th[1] / 2.0; d[2] = th[2] / 2.0; d[3] = 1.0; }
  else { const double s = std::sin(n / 2.0); for (int k = 0; k < 3; k++) d[k] = th[k] / n * s; d[3] = std::cos(n / 2.0); }
  const double o[4] = {qi[3] * d[0] + qi[0] * d[3] + qi[1] * d[2] - qi[2] * d[1], qi[3] * d[1] - qi[0] * d[2] + qi[1] * d[3] + qi[2] * d[0],
                       qi[3] * d[2] + qi[0] * d[1] - qi[1] * d[0] + qi[2] * d[3], qi[3] * d[3] - qi[0] * d[0] - qi[1] * d[1] - qi[2] * d[2]};
  chart_unit(o, q);
}

// the pose records in the retraction's layout [p, q, 0]: the chart's attitudes composed and normalised
static std::vector<double> chart_poses(const d2pgo_handle *h) {
  std::vector<double> out(h->poses.size(), 0.0);
  for (size_t i = 0; i < h->ids.size(); i++) {
    memcpy(&out[i * 8], &h->poses[i * 8], 24);
    chart_attitude(&h->poses[i * 8], &h->chart_qinit[i * 4], &out[i * 8 + 3]);
  }
  return out;
}

static int chart_get_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, double *out) {
  if (n < 0 || (n > 0 && (!ids || !out))) return pgo_fail(h, 1, "get_poses: null argument or negative count");
  for (int k = 0; k < n; k++) {
    auto it = h->index.find(ids[k]);
    if (it == h->index.end()) return pgo_fail(h, 2, "get_poses: unknown id");
    const size_t i = (size_t)it->second;
    memcpy(out + (size_t)k * 7, &h->poses[i * 8], 24);
    chart_attitude(&h->poses[i * 8], &h->chart_qinit[i * 4], out + (size_t)k * 7 + 3);
  }
  return 0;
}

// d2pgo_set_poses on a chart handle: ids already present keep their [p, theta] and q_init, new ids start at [p, 0] with q_init
// = their normalised attitude (PGOState::addFrame)
static int chart_set_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses7, const uint8_t *fixed) {
  std::vector<double> x((size_t)n * 7, 0.0), qi((size_t)n * 4);
  std::unordered_map<int64_t, int> seen;
  for (int k = 0; k < n; k++) {
    if (!seen.emplace(ids[k], k).second) return pgo_fail(h, 2, "set_poses: duplicate pose id");
    auto it = h->index.find(ids[k]);
    if (it != h->index.end()) {
      memcpy(&x[(size_t)k * 7], &h->poses[(size_t)it->second * 8], 48);
      memcpy(&qi[(size_t)k * 4], &h->chart_qinit[(size_t)it->second * 4], 32);
      continue;
    }
    const double *p = poses7 + (size_t)k * 7;
    if (!all_finite(p, 7) || !chart_unit(p + 3, &qi[(size_t)k * 4]))
      return pgo_fail(h, 2, "set_poses: pose id " + std::to_string(ids[k]) + ": non-finite value or zero quaternion (the perturbation chart takes its q_init from it)");
    memcpy(&x[(size_t)k * 7], p, 24);
  }
  if (int rc = pgo_set_poses(h, n, ids, x.data(), 7, fixed, "set_poses")) return rc;
  h->chart_qinit.swap(qi);
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
  h->own_stream = true;
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  *out = h;
  return 0;
}

int d2pgo_destroy(d2pgo_handle *h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device);
  cudaStreamSynchronize(h->stream);
  if (h->comm) nccl_comm_destroy(h->comm);
  delete h;
  return 0;
}

const char *d2pgo_last_error(const d2pgo_handle *h) { return h ? h->err.c_str() : "null handle"; }

int d2pgo_set_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *poses7, const uint8_t *fixed) {
  if (!h || n <= 0) return 1;
  if (int rc = pgo_want_dof(h, 6, "set_poses")) return rc;
  if (h->chart) return chart_set_poses(h, n, ids, poses7, fixed);
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
  if (h->arock) { h->err = "comm_init: the handle is in ARock mode (each agent solves its own sub-graph; edge sharding splits one graph)"; return 5; }
  if (h->chart) { h->err = "comm_init: the handle is in the perturbation chart, which has no edge-sharded form (d2pgo_set_chart(h, D2PGO_CHART_RETRACTION, ...) first)"; return 5; }
  if (h->linear_solver == D2PGO_LINEAR_SPARSE_CHOLESKY) { h->err = "comm_init: the handle solves with the sparse Cholesky, which has no edge-sharded form (d2pgo_set_linear_solver PCG first)"; return 5; }
  cudaSetDevice(h->cfg.device);
  if (nccl_comm_init(&h->comm, unique_id, rank, nranks, h->err)) return 3;
  h->rank = rank; h->nranks = nranks;
  return 0;
}

}  // extern "C"

// per-block cost partials of the edges, the gravity priors and the synced duals, in that order
static int pgo_alloc_cost_part(d2pgo_handle *h) {
  const size_t nbe = (h->ea.size() + 127) / 128, nbg = (h->gp_pose.size() + 127) / 128, nbk = (size_t)(std::max(h->ak_n, 0) + 127) / 128;
  PCK(h->d_cost_part.alloc(nbe + nbg + nbk + 1));
  return 0;
}

static int pgo_upload(d2pgo_handle *h) {
  const size_t N = h->ids.size(), E = h->ea.size(), nbp = (N + 127) / 128;
  const size_t D = h->dof, DD = D * D;
  for (int b = 0; b < 2; b++) { PCK(h->d_x[b].alloc(N * 8)); PCK(h->d_g[b].alloc(N * D)); PCK(h->d_D[b].alloc(N * DD)); PCK(h->d_lin[b].alloc(E * (D + 2 * DD))); }
  PCK(h->d_rel.alloc(E * 8)); PCK(h->d_sinfo.alloc(E * DD)); PCK(h->d_Minv.alloc(N * DD));
  PCK(h->d_dx.alloc(N * D)); PCK(h->d_r.alloc(N * D)); PCK(h->d_z.alloc(N * D)); PCK(h->d_p.alloc(N * D)); PCK(h->d_Ap.alloc(N * D)); PCK(h->d_cost.alloc(2));
  const size_t G = h->gp_pose.size();
  PCK(h->d_damp.alloc(N * D)); PCK(h->d_t.alloc(E * 2 * D)); PCK(h->d_part.alloc(5 * nbp));
  if (int rc = pgo_alloc_cost_part(h)) return rc;
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
  if (h->chart == D2PGO_CHART_PERTURB) {
    PCK(h->d_qinit.alloc(N * 4));
    PCK(cudaMemcpyAsync(h->d_qinit.p, h->chart_qinit.data(), N * 32, cudaMemcpyHostToDevice, h->stream));
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
  PgoPriorDev pr; memset(&pr, 0, sizeof pr);
  pr.n_prior = (int)h->gp_pose.size(); pr.pose = h->d_gp_pose.p; pr.prior_of = h->d_prior_of.p; pr.u = h->d_gp_u.p; pr.S = h->d_gp_S.p; pr.lin = h->d_glin[cur].p;
  return pr;
}

static PgoArockDev pgo_arock_view(d2pgo_handle *h, int cur) {
  PgoArockDev a; memset(&a, 0, sizeof a);
  a.n_dual = h->ak_n > 0 ? h->ak_n : 0; a.pose = h->d_ak_pose.p; a.ptr = h->d_ak_ptr.p; a.of = h->d_ak_of.p; a.yr = h->d_ak_yr.p; a.yl = h->d_ak_yl.p;
  a.qinit = h->d_ak_qinit.p; a.lin = h->d_ak_lin[cur].p;
  const bool six = h->dof == 6;
  a.wT = six ? std::sqrt(h->acfg.rho_frame_T) : h->acfg.rho_frame_T; a.wR = six ? std::sqrt(h->acfg.rho_frame_theta) : h->acfg.rho_frame_theta;
  a.eta = h->acfg.eta_k;
  return a;
}

template <class F> static int with_policy(d2pgo_handle *h, F &&f) {   // f(the policy of the handle's parameterisation)
  return h->dof == 4 ? f(PgoRetraction<PgoEdge4>()) : h->chart ? f(PgoChart6()) : f(PgoRetraction<PgoEdge6>());
}

// cost (+ lin records, gradient, block diagonal of buffer `b`) at pose buffer `b`; all-reduced across the ranks.  grav: the
// gravity priors of this rank (6-DoF only; their cost partials follow the edges', their terms enter g and D after each pose's
// edges).  ark: the ARock proximal terms of the synced dual table (cost partials last, g and D after the edges and priors).
// the kernels of one linearisation of buffer b on stream st, the total cost into *cost_dev
template <class H>
static void pgo_linearize_enqueue(d2pgo_handle *h, cudaStream_t st, int b, int want_jac, bool grav, bool ark, double *cost_dev) {
  using K = typename H::Kern;
  PgoDev d = pgo_view(h, b);
  const PgoPriorDev pr = pgo_prior_view(h, b);
  const PgoArockDev ak = pgo_arock_view(h, b);
  const int nbe = (d.n_edge + 127) / 128, nbg = grav ? (pr.n_prior + 127) / 128 : 0, nbk = ark ? (ak.n_dual + 127) / 128 : 0;
  if (d.n_edge > 0) H::lin_edges(h, st, d, h->d_cost_part.p, want_jac);
  if (nbg > 0) H::lin_priors(h, st, d, pr, h->d_cost_part.p + nbe, want_jac);
  if (nbk > 0) H::lin_arock(st, d, ak, h->d_cost_part.p + nbe + nbg);
  k_pgo_sum<<<1, 128, 0, st>>>(h->d_cost_part.p, nbe + nbg + nbk, cost_dev);
  if (want_jac && grav) {
    if constexpr (kPriorKern<K>) k_pgo_gD<K, true><<<d.nbp, 128, 0, st>>>(d, h->d_g[b].p, h->d_D[b].p, pr);
  } else if (want_jac) k_pgo_gD<K, false><<<d.nbp, 128, 0, st>>>(d, h->d_g[b].p, h->d_D[b].p, pr);
  if (want_jac && nbk > 0) k_pgo_arock_gD<H::D><<<d.nbp, 128, 0, st>>>(d, h->d_g[b].p, h->d_D[b].p, ak);
}

template <class H>
static int pgo_linearize(d2pgo_handle *h, int b, int want_jac, bool grav, bool ark, double *cost) {
  constexpr int D = H::D;
  const size_t N = h->ids.size();
  pgo_linearize_enqueue<H>(h, h->stream, b, want_jac, grav, ark, h->d_cost.p);
  if (h->comm) {
    if (nccl_allreduce_f64(h->comm, h->d_cost.p, 1, h->stream)) { h->err = "ncclAllReduce(cost) failed"; return 40; }
    if (want_jac && (nccl_allreduce_f64(h->comm, h->d_g[b].p, N * D, h->stream) || nccl_allreduce_f64(h->comm, h->d_D[b].p, N * D * D, h->stream))) { h->err = "ncclAllReduce(g, D) failed"; return 40; }
  }
  PCK(cudaMemcpyAsync(cost, h->d_cost.p, 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  return 0;
}

constexpr int kCgChunk = 16;   // CG iterations between two looks at the convergence flag (one graph launch on a single rank)

// the pose pass of one CG iteration, with the gravity priors' terms when grav (6-DoF only)
template <class P, bool LOCAL>
static void pgo_cg_pose(d2pgo_handle *h, const PgoDev &d, int par, double tol2, const PgoPriorDev &pr, bool grav) {
  if constexpr (kPriorKern<P>) {
    if (grav) { k_pgo_cg_pose<P, LOCAL, true><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2, pr); return; }
  }
  k_pgo_cg_pose<P, LOCAL, false><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2, pr);
}

// n CG iterations (n <= kCgChunk, the chunk starting at an iteration index that is a multiple of kCgChunk, so k & 1 is the
// global parity); ark: the proximal terms' damping pass.  The rotation rows (PgoRotRow) solve on one rank without proximal
// terms, so only their single-rank kernels exist.
template <class P>
static int pgo_cg_chunk(d2pgo_handle *h, const PgoDev &d, const PgoPriorDev &pr, const PgoArockDev &ak, double tol2, bool grav, bool ark, int n) {
  const int ge = (d.n_edge + 127) / 128;
  for (int k = 0; k < n; k++) {
    const int par = k & 1;
    if (d.n_edge > 0) k_pgo_cg_edge<P><<<ge, 128, 0, h->stream>>>(d, par, tol2);
    if (!ark && !h->comm) {
      pgo_cg_pose<P, false>(h, d, par, tol2, pr, grav);
    } else if constexpr (!std::is_same<P, PgoRotRow>::value) {
      pgo_cg_pose<P, true>(h, d, par, tol2, pr, grav);
      if (ark) {   // an ARock handle has no communicator (d2pgo_comm_init refuses it)
        k_pgo_arock_cg_pAp<P><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2, ak);
      } else {
        // every rank holds the same r, z, p (the all-reduced products are bitwise identical), so all of them reach the same
        // `done` decision at the same iteration and the collective below is always matched
        if (nccl_allreduce_f64(h->comm, d.Ap, (size_t)d.n_pose * P::D, h->stream)) { h->err = "ncclAllReduce(Ap) failed"; return 40; }
        k_pgo_cg_pAp<P><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2);
      }
    }
    k_pgo_cg_step<P><<<d.nbp, 128, 0, h->stream>>>(d, par, tol2);
  }
  return 0;
}

// (J^T J + lambda diag D) dx = -g at linearisation buffer `cur` by block-Jacobi preconditioned CG (J^T J is never formed), in
// chunks of kCgChunk iterations, the last one shortened so that at most max_it iterations run, until the convergence flag; *s
// holds the CG scalars after the last chunk.  On a single rank a chunk is one launch of one of the buffer's two captured graphs
// (full chunk, short last chunk).  A graph's kernel nodes hold the arguments they were captured with (pointers, counts,
// weights, tol2) and its length, so it is captured again whenever any of those bytes differ.
template <class P>
static int pgo_pcg(d2pgo_handle *h, int cur, double lambda, double tol2, int max_it, bool grav, bool ark, PgoScalars *s) {
  const PgoDev d = pgo_view(h, cur);
  const PgoPriorDev pr = pgo_prior_view(h, cur);
  const PgoArockDev ak = pgo_arock_view(h, cur);
  k_pgo_precond<P><<<d.nbp, 128, 0, h->stream>>>(d, h->d_D[cur].p, lambda);
  k_pgo_cg_init<P><<<d.nbp, 128, 0, h->stream>>>(d, h->d_g[cur].p);
  k_pgo_cg_init2<<<1, 128, 0, h->stream>>>(d);
  std::string args((const char *)&d, sizeof d);
  args.append((const char *)&pr, sizeof pr).append((const char *)&ak, sizeof ak).append((const char *)&tol2, sizeof tol2);
  args += (char)grav; args += (char)ark;
  for (int k = 0; k < max_it; k += kCgChunk) {
    const int n = std::min(kCgChunk, max_it - k);
    if (h->comm) {
      if (int rc = pgo_cg_chunk<P>(h, d, pr, ak, tol2, grav, ark, n)) return rc;
    } else {
      const int which = n < kCgChunk;
      cudaGraphExec_t &graph = h->cg_graph[cur][which];
      const std::string key = args + std::string((const char *)&n, sizeof n);
      if (!graph || h->cg_args[cur][which] != key) {
        if (graph) { cudaGraphExecDestroy(graph); graph = nullptr; }
        cudaGraph_t g;
        PCK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
        pgo_cg_chunk<P>(h, d, pr, ak, tol2, grav, ark, n);
        PCK(cudaStreamEndCapture(h->stream, &g));
        PCK(cudaGraphInstantiate(&graph, g, 0));
        cudaGraphDestroy(g);
        h->cg_args[cur][which] = key;
      }
      PCK(cudaGraphLaunch(graph, h->stream));
    }
    PCK(cudaMemcpyAsync(s, h->d_s.p, sizeof *s, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
    if (s->done) break;   // identical on every rank (see pgo_cg_chunk)
  }
  return 0;
}

// the sparse Cholesky's symbolic analysis of the handle's current structure (host only: poses, fixed flags, edge ends), redone
// when that structure changed; then the size limits, before any device work of the solve
static int pgo_chol_analyse(d2pgo_handle *h) {
  if (!h->chol) h->chol.reset(new d2pgo_chol::Numeric());
  d2pgo_chol::Symbolic &S = h->chol->sym;
  if (S.D == h->dof && S.fixed == h->fixed && S.ea == h->ea && S.eb == h->eb) return 0;
  h->chol->release();
  if (int rc = d2pgo_chol::analyse((int)h->ids.size(), h->fixed.data(), (int)h->ea.size(), h->ea.data(), h->eb.data(), h->dof, S, h->err)) {
    S = d2pgo_chol::Symbolic();
    return rc;
  }
  return 0;
}

static int pgo_chol_prepare(d2pgo_handle *h) {
  if (int rc = pgo_chol_analyse(h)) return rc;
  const d2pgo_chol::Symbolic &S = h->chol->sym;
  size_t free_b = 0, total_b = 0;
  PCK(cudaMemGetInfo(&free_b, &total_b));
  if (!h->chol->dev_ready) {
    const std::string why = d2pgo_chol::check_limits(S, free_b);
    if (!why.empty()) { h->err = why; return 7; }
  }
  return 0;
}

// one exact step (J^T J + lambda diag D + 1e-12) dx = -g at linearisation buffer `cur` into d_dx
static int pgo_chol_step(d2pgo_handle *h, int cur, double lambda, bool *failed) {
  d2pgo_chol::Numeric &c = *h->chol;
  if (!c.dev_ready) if (int rc = c.upload(h->stream, h->err)) return rc;
  const d2pgo_chol::Lin in{h->d_lin[cur].p, h->d_D[cur].p, h->d_g[cur].p, h->d_fixed.p, h->d_ea.p, h->d_eb.p, h->d_dx.p};
  return c.step(h->stream, cur, in, lambda, failed, h->err);
}

// the LM loop in the pose parameterisation H, with the handle's gravity priors and, when ark, the ARock proximal terms of the
// synced dual table
template <class H>
static int pgo_solve(d2pgo_handle *h, d2pgo_report *rep, bool ark) {
  int rc;
  const bool chol = h->linear_solver == D2PGO_LINEAR_SPARSE_CHOLESKY, grav = !h->gp_pose.empty();
  if (chol) {
    if ((rc = pgo_chol_prepare(h))) return rc;
    h->chol->factorizations = h->chol->failed = 0; h->chol->factor_ms = h->chol->solve_ms = 0.0;
  }
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  const int N = (int)h->ids.size();
  d2pgo_report R; memset(&R, 0, sizeof R);
  PCK(cudaEventRecord(h->ev0, h->stream));
  int cur = 0;                    // buffer (poses, lin records, g, D) of the accepted point
  double cost = 0, lambda = h->cfg.lambda0;
  if ((rc = pgo_linearize<H>(h, cur, 1, grav, ark, &cost))) return rc;
  R.initial_cost = cost;
  const double tol2 = h->cfg.pcg_tolerance * h->cfg.pcg_tolerance;
  for (int it = 0; it < h->cfg.max_iterations; it++) {
    PgoScalars s; memset(&s, 0, sizeof s);
    if (chol) {   // the exact step from the sparse Cholesky; a failed factorisation is a rejected step
      bool failed = false;
      if ((rc = pgo_chol_step(h, cur, lambda, &failed))) return rc;
      if (failed) {
        R.iterations++;
        lambda = lambda > 0 ? lambda * 4.0 : 1e-4;
        if (lambda > 1e8) break;
        continue;
      }
    } else if ((rc = pgo_pcg<typename H::Kern>(h, cur, lambda, tol2, h->cfg.pcg_max_iterations, grav, ark, &s))) return rc;
    H::retract(h->stream, pgo_view(h, cur), h->d_x[1 - cur].p);
    double cand = 0;
    if ((rc = pgo_linearize<H>(h, 1 - cur, 1, grav, ark, &cand))) return rc;
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
  if (cur != 0) PCK(cudaMemcpyAsync(h->d_x[0].p, h->d_x[1].p, (size_t)N * 64, cudaMemcpyDeviceToDevice, h->stream));   // a following solve starts from buffer 0
  PCK(cudaMemcpyAsync(h->poses.data(), h->d_x[cur].p, (size_t)N * 64, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  R.final_cost = cost; R.device_ms = ms;
  if (rep) *rep = R;
  return 0;
}

// ---- the ceres minimiser's host side: refusals, the graph of one solve, and the solve.  The graph:
//   k_lm_start, linearisation of x0 (buffer 0), k_lm_scale, k_lm_xnorm, then WHILE(loop) {
//     k_lm_begin; IF(go) { factor + solve (k_chol_diag_lm's damping), k_lm_model, k_lm_mid;
//                          IF(eval) { x1 = x0 [+] dx, cost of buffer 1 into d_cost[1] }; k_lm_end;
//                          IF(accept) { x0 <- x1 (N x 64 bytes), linearisation of x0 into d_cost[0], k_lm_xnorm } } }
// Accepting copies the candidate's poses into buffer 0 and relinearises there (as ceres evaluates the Jacobian at the new x),
// so the kernels' buffer pointers are fixed and the graph serves every solve of the same buffers.
static int lm_refuse(d2pgo_handle *h, const char *what) {
  if (h->minimizer != D2PGO_MINIMIZER_CERES_LM) return 0;
  if (h->comm) return pgo_fail(h, 5, std::string(what) + ": the ceres minimiser has no edge-sharded form (the handle has a communicator)");
  if (h->linear_solver != D2PGO_LINEAR_SPARSE_CHOLESKY)
    return pgo_fail(h, 5, std::string(what) + ": the ceres minimiser takes exact steps from the sparse Cholesky (d2pgo_set_linear_solver(h, D2PGO_LINEAR_SPARSE_CHOLESKY) first)");
  if (!h->driver_version && cudaDriverGetVersion(&h->driver_version) != cudaSuccess) h->driver_version = 0;
  if (h->driver_version < 12040)
    return pgo_fail(h, 3, std::string(what) + ": the ceres minimiser runs as one CUDA graph with conditional nodes, which needs a driver for CUDA 12.4 or newer (this one: " +
                              std::to_string(h->driver_version) + ")");
  return 0;
}

// appends a conditional node on the handle `c` after the work captured so far on st; *body = the graph it runs
static cudaError_t lm_cond(cudaStream_t st, cudaGraphConditionalHandle c, cudaGraphConditionalNodeType type, cudaGraph_t *body) {
  cudaStreamCaptureStatus cs;
  cudaGraph_t g;
  const cudaGraphNode_t *deps = nullptr;
  size_t nd = 0;
  cudaError_t e = cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &nd);
  if (e != cudaSuccess) return e;
  cudaGraphNodeParams p = {cudaGraphNodeTypeConditional};
  p.conditional.handle = c; p.conditional.type = type; p.conditional.size = 1;
  cudaGraphNode_t node;
  if ((e = cudaGraphAddNode(&node, g, deps, nd, &p)) != cudaSuccess) return e;
  *body = p.conditional.phGraph_out[0];
  return cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies);
}

template <class H>
static int lm_build(d2pgo_handle *h, bool grav, bool ark, cudaStream_t *cs) {
  const PgoDev d0 = pgo_view(h, 0), d1 = pgo_view(h, 1);
  const PgoPriorDev pr = pgo_prior_view(h, 0);
  const PgoArockDev ak = pgo_arock_view(h, 0);
  const int nbp = d0.nbp, nbe = (d0.n_edge + 127) / 128, nbg = grav ? (pr.n_prior + 127) / 128 : 0, nbk = ark ? (ak.n_dual + 127) / 128 : 0;
  const int nbm = nbe + nbg + nbk + nbp;
  const d2pgo_lm::View v{H::D, d0.n_pose, d0.n_edge, grav ? pr.n_prior : 0, ark ? ak.n_dual : 0, d0.x, h->d_g[0].p, d0.dx, d0.lin, pr.lin, ak.lin,
                         d0.fixed, d0.ea, d0.eb, pr.pose, ak.pose};
  LmState *s = h->d_lm.p;
  double *xpart = h->d_lm_part.p, *mpart = xpart + 2 * (size_t)nbp, *cost = h->d_cost.p;
  d2pgo_minimizer_iteration *trace = h->d_lm_trace.p;
  const d2pgo_chol::Lin in{h->d_lin[0].p, h->d_D[0].p, h->d_g[0].p, h->d_fixed.p, h->d_ea.p, h->d_eb.p, h->d_dx.p};
  const d2pgo_chol::LmDamping dm{h->d_lm_scale.p, &s->radius};
  cudaGraph_t top = nullptr, body, go_g, eval_g, acc_g;
  cudaGraphConditionalHandle loop, go, eval, acc;
  PCK(cudaGraphCreate(&top, 0));
  std::unique_ptr<CUgraph_st, cudaError_t (*)(cudaGraph_t)> own(top, cudaGraphDestroy);
  const cudaStreamCaptureMode mode = cudaStreamCaptureModeThreadLocal;
  PCK(cudaGraphConditionalHandleCreate(&loop, top, 1, cudaGraphCondAssignDefault));
  PCK(cudaStreamBeginCaptureToGraph(cs[0], top, nullptr, nullptr, 0, mode));
  d2pgo_lm::start(cs[0], s);
  pgo_linearize_enqueue<H>(h, cs[0], 0, 1, grav, ark, cost);
  d2pgo_lm::scale(cs[0], v, h->d_D[0].p, s, h->d_lm_scale.p);
  H::xnorm(cs[0], v, xpart);
  PCK(lm_cond(cs[0], loop, cudaGraphCondTypeWhile, &body));
  PCK(cudaStreamEndCapture(cs[0], &top));
  PCK(cudaGraphConditionalHandleCreate(&go, body, 0, 0));
  PCK(cudaStreamBeginCaptureToGraph(cs[1], body, nullptr, nullptr, 0, mode));
  d2pgo_lm::begin(cs[1], s, cost, xpart, nbp, loop, go);
  PCK(lm_cond(cs[1], go, cudaGraphCondTypeIf, &go_g));
  PCK(cudaStreamEndCapture(cs[1], &body));
  PCK(cudaGraphConditionalHandleCreate(&eval, go_g, 0, 0));
  PCK(cudaGraphConditionalHandleCreate(&acc, go_g, 0, 0));
  PCK(cudaStreamBeginCaptureToGraph(cs[2], go_g, nullptr, nullptr, 0, mode));
  if (int rc = h->chol->enqueue_lm(cs[2], in, dm, h->err)) { cudaStreamEndCapture(cs[2], &go_g); return rc; }
  d2pgo_lm::model(cs[2], v, nbe, nbg, nbk, mpart);
  d2pgo_lm::mid(cs[2], s, h->chol->d_fail, mpart, nbm, trace, eval);
  PCK(lm_cond(cs[2], eval, cudaGraphCondTypeIf, &eval_g));
  d2pgo_lm::end(cs[2], s, cost, trace, acc);
  PCK(lm_cond(cs[2], acc, cudaGraphCondTypeIf, &acc_g));
  PCK(cudaStreamEndCapture(cs[2], &go_g));
  PCK(cudaStreamBeginCaptureToGraph(cs[3], eval_g, nullptr, nullptr, 0, mode));
  H::retract(cs[3], d0, h->d_x[1].p);
  pgo_linearize_enqueue<H>(h, cs[3], 1, 0, grav, ark, cost + 1);
  PCK(cudaStreamEndCapture(cs[3], &eval_g));
  PCK(cudaStreamBeginCaptureToGraph(cs[3], acc_g, nullptr, nullptr, 0, mode));
  PCK(cudaMemcpyAsync(h->d_x[0].p, d1.x, (size_t)d0.n_pose * 64, cudaMemcpyDeviceToDevice, cs[3]));
  pgo_linearize_enqueue<H>(h, cs[3], 0, 1, grav, ark, cost);
  H::xnorm(cs[3], v, xpart);
  PCK(cudaStreamEndCapture(cs[3], &acc_g));
  PCK(cudaGetLastError());
  if (h->lm_graph) { cudaGraphExecDestroy(h->lm_graph); h->lm_graph = nullptr; }
  PCK(cudaGraphInstantiate(&h->lm_graph, top, 0));
  return 0;
}

constexpr int kLmTraceCap = 16384;   // trace records kept per solve (the first iterations)

// ceres' TrustRegionMinimizer with LevenbergMarquardtStrategy (d2pgo_set_minimizer): one graph launch, one synchronisation
template <class H>
static int pgo_solve_ceres(d2pgo_handle *h, d2pgo_report *rep, bool ark) {
  int rc, syncs = 1;
  if ((rc = pgo_chol_prepare(h))) return rc;
  if (!h->uploaded) { if ((rc = pgo_upload(h))) return rc; syncs++; }
  if (!h->chol->dev_ready) { if ((rc = h->chol->upload(h->stream, h->err))) return rc; syncs++; }
  const bool grav = !h->gp_pose.empty();
  const d2pgo_ceres_lm_config &c = h->lm_cfg;
  const int N = (int)h->ids.size(), D = H::D, nbp = (N + 127) / 128;
  const int nbm = (int)(h->ea.size() + 127) / 128 + (grav ? (int)(h->gp_pose.size() + 127) / 128 : 0) + (ark ? (std::max(h->ak_n, 0) + 127) / 128 : 0) + nbp;
  const int cap = std::max(1, std::min(c.max_num_iterations, kLmTraceCap));
  PCK(h->d_lm.alloc(1)); PCK(h->d_lm_scale.alloc((size_t)N * D)); PCK(h->d_lm_part.alloc(2 * (size_t)nbp + 3 * (size_t)nbm));
  PCK(h->d_lm_trace.alloc(cap));
  // the graph holds every pointer and count its kernels were captured with: rebuilt when any of those bytes differ
  std::string key;
  auto put = [&key](const void *p, size_t n) { key.append((const char *)p, n); };
  for (int b = 0; b < 2; b++) {
    const PgoDev d = pgo_view(h, b); const PgoPriorDev pr = pgo_prior_view(h, b); const PgoArockDev ak = pgo_arock_view(h, b);
    put(&d, sizeof d); put(&pr, sizeof pr); put(&ak, sizeof ak);
  }
  const void *ptrs[8] = {h->d_lm.p, h->d_lm_scale.p, h->d_lm_part.p, h->d_lm_trace.p, h->d_cost.p, h->d_cost_part.p, h->chol.get(), h->d_qinit.p};
  const int gen[4] = {h->chol->generation, grav, ark, h->chart};
  put(ptrs, sizeof ptrs); put(gen, sizeof gen);
  if (!h->lm_graph || h->lm_key != key) {
    cudaStream_t cs[4] = {h->stream, nullptr, nullptr, nullptr};
    for (int k = 1; k < 4; k++) PCK(cudaStreamCreateWithFlags(&cs[k], cudaStreamNonBlocking));
    rc = lm_build<H>(h, grav, ark, cs);
    for (int k = 1; k < 4; k++) cudaStreamDestroy(cs[k]);
    if (rc) { h->lm_key.clear(); return rc; }
    h->lm_key = key;
  }
  LmState st;
  memset(&st, 0, sizeof st);
  st.radius0 = c.initial_trust_region_radius; st.max_radius = c.max_trust_region_radius; st.min_radius = c.min_trust_region_radius;
  st.min_diag = c.min_lm_diagonal; st.max_diag = c.max_lm_diagonal; st.min_rel_dec = c.min_relative_decrease;
  st.ftol = c.function_tolerance; st.gtol = c.gradient_tolerance; st.ptol = c.parameter_tolerance; st.budget_s = c.max_solver_time_in_seconds;
  st.max_iter = c.max_num_iterations; st.max_invalid = c.max_num_consecutive_invalid_steps; st.jacobi = c.jacobi_scaling; st.trace_cap = cap;
  PCK(cudaMemcpyAsync(h->d_lm.p, &st, sizeof st, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaEventRecord(h->ev0, h->stream));
  PCK(cudaGraphLaunch(h->lm_graph, h->stream));
  PCK(cudaEventRecord(h->ev1, h->stream));
  PCK(cudaMemcpyAsync(h->poses.data(), h->d_x[0].p, (size_t)N * 64, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaMemcpyAsync(&st, h->d_lm.p, sizeof st, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));   // the solve's one synchronisation
  float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  d2pgo_minimizer_summary &m = h->lm_report;
  memset(&m, 0, sizeof m);
  m.termination_type = st.type; m.reason = st.reason; m.successful_steps = st.ok; m.unsuccessful_steps = st.bad; m.host_syncs = syncs;
  m.final_radius = st.radius; m.elapsed_s = (double)(st.t_end - st.t0) * 1e-9; m.initial_cost = st.cost0; m.final_cost = st.cost;
  h->lm_ran = true; h->lm_trace_n = std::min(st.iter, cap);
  h->chol->factorizations = st.iter; h->chol->failed = st.pivot_fail; h->chol->factor_ms = h->chol->solve_ms = 0.0;
  d2pgo_report R; memset(&R, 0, sizeof R);
  R.iterations = st.ok + st.bad; R.accepted = st.ok; R.converged = st.type == D2PGO_TERMINATION_CONVERGENCE;
  R.initial_cost = st.cost0; R.final_cost = st.cost; R.device_ms = ms;
  if (rep) *rep = R;
  return 0;
}

// the handle's minimiser (d2pgo_set_minimizer); its refusals (lm_refuse) come before any state changes, in the callers
template <class H>
static int pgo_minimize(d2pgo_handle *h, d2pgo_report *rep, bool ark) {
  h->lm_ran = false;
  return h->minimizer == D2PGO_MINIMIZER_CERES_LM ? pgo_solve_ceres<H>(h, rep, ark) : pgo_solve<H>(h, rep, ark);
}

extern "C" {

int d2pgo_solve(d2pgo_handle *h, d2pgo_report *rep) {
  if (!h || h->ids.empty()) return 1;
  if (int rc = lm_refuse(h, "solve")) return rc;
  cudaSetDevice(h->cfg.device);
  return with_policy(h, [&](auto pol) { return pgo_minimize<decltype(pol)>(h, rep, false); });
}

int d2pgo_get_poses(d2pgo_handle *h, int32_t n, const int64_t *ids, double *out) {
  if (!h) return 1;
  if (int rc = pgo_want_dof(h, 6, "get_poses")) return rc;
  if (h->chart) return chart_get_poses(h, n, ids, out);
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
  if ((rc = with_policy(h, [&](auto pol) { return pgo_linearize<decltype(pol)>(h, 0, 1, false, false, &cost); }))) return rc;
  std::vector<double> tmp(E * W);
  PCK(cudaMemcpyAsync(tmp.data(), h->d_lin[0].p, E * W * 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
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
  if ((rc = with_policy(h, [&](auto pol) { return pgo_linearize<decltype(pol)>(h, 0, 1, true, false, &cost); }))) return rc;
  std::vector<double> tmp(G * 12);
  PCK(cudaMemcpyAsync(tmp.data(), h->d_glin[0].p, G * 12 * 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  for (size_t k = 0; k < G; k++) {   // device layout is field-major [12][G]: r(3), J_theta (3x3)
    double *o = out + k * 21;
    for (int a = 0; a < 3; a++) o[a] = tmp[a * G + k];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 6; b++) o[3 + a * 6 + b] = b < 3 ? 0.0 : tmp[(3 + a * 3 + b - 3) * G + k];
  }
  return 0;
}

}  // extern "C"

// ---- ARock host side

// poses the local problem uses: those an edge or a gravity prior touches (ARockSolver::all_estimating_params)
static std::vector<char> arock_in_problem(const d2pgo_handle *h) {
  std::vector<char> in(h->ids.size(), 0);
  for (size_t e = 0; e < h->ea.size(); e++) in[h->ea[e]] = in[h->eb[e]] = 1;
  for (int p : h->gp_pose) in[p] = 1;
  return in;
}

// ---- the ARock dual tables (d2pgo_handle::pose_table, rot_table): what the pose and the rotation exchanges share
using d2pgo_host::ArockDuals;
using d2pgo_host::ArockTable;

// a received message, before it is queued: counts and pointers, its dual width D, not from this agent, finite, no frame twice
static int arock_receive_check(d2pgo_handle *h, const char *what, int D, int32_t sender, int32_t n, const int64_t *frame_ids,
                               int32_t dim, const double *duals) {
  const std::string w(what);
  if (n < 0 || (n > 0 && (!frame_ids || !duals))) return pgo_fail(h, 1, w + ": null argument or negative count");
  if (dim != D) return pgo_fail(h, 2, w + ": duals of dimension " + std::to_string(dim) + ", this exchange's duals have " + std::to_string(D));
  if (sender == h->acfg.self_id) return pgo_fail(h, 2, w + ": a message from this agent itself (self_id " + std::to_string(sender) + ")");
  if (!all_finite(duals, (size_t)n * dim)) return pgo_fail(h, 2, w + ": non-finite dual");
  std::unordered_map<int64_t, int> seen;
  for (int k = 0; k < n; k++) if (!seen.emplace(frame_ids[k], k).second) return pgo_fail(h, 2, w + ": frame id " + std::to_string(frame_ids[k]) + " twice in one message");
  return 0;
}

template <int W> static void arock_queue(ArockTable<W> &t, int32_t sender, int32_t target, int32_t n, const int64_t *frame_ids, int D, const double *duals) {
  t.inbox.push_back(d2pgo_host::ArockMsg{sender, target, std::vector<int64_t>(frame_ids, frame_ids + n), std::vector<double>(duals, duals + (size_t)n * D)});
}

// receiveAll / processPGOData (ARockPGO.cpp:13-70; rotation_initialization_arock.hpp:104-111, :142-182): t's messages applied to
// duals in arrival order.  A frame counts only if the local problem contains it (in[pose index]); the message applies if
// target == self or there is no dual (sender, f) yet: a new dual takes the value on both sides, an existing one on y_r only.
template <int W>
static void arock_apply_inbox(const d2pgo_handle *h, const ArockTable<W> &t, const std::vector<char> &in, int D, ArockDuals<W> &duals) {
  for (const auto &m : t.inbox)
    for (size_t k = 0; k < m.frames.size(); k++) {
      auto it = h->index.find(m.frames[k]);
      if (it == h->index.end() || !in[it->second]) continue;
      const auto key = std::make_pair(m.sender, m.frames[k]);
      auto d = duals.find(key);
      if (m.target != h->acfg.self_id && d != duals.end()) continue;
      const double *v = &m.duals[k * D];
      if (d == duals.end()) { d2pgo_host::ArockDual<W> nd; memset(&nd, 0, sizeof nd); memcpy(nd.yl, v, D * 8); memcpy(nd.yr, v, D * 8); duals.emplace(key, nd); }
      else memcpy(d->second.yr, v, D * 8);
    }
}

// the duals [lo, hi) in table order: y_l [n][D] and (if not null) y_r [n][D]; and back, y_l only
template <class It> static void arock_flatten(It lo, It hi, int D, double *yl, double *yr) {
  for (size_t k = 0; lo != hi; ++lo, ++k) {
    memcpy(yl + k * D, lo->second.yl, D * 8);
    if (yr) memcpy(yr + k * D, lo->second.yr, D * 8);
  }
}
template <int W> static void arock_set_yl(ArockDuals<W> &duals, int D, const double *yl) {
  size_t k = 0;
  for (auto &kv : duals) memcpy(kv.second.yl, yl + k++ * D, D * 8);
}

// the neighbours of the table, ascending
template <int W> static int arock_neighbours(d2pgo_handle *h, const ArockTable<W> &t, const char *what, int32_t max_n, int32_t *n_out, int32_t *ids_out) {
  if (!n_out || max_n < 0 || (max_n > 0 && !ids_out)) return pgo_fail(h, 1, std::string(what) + ": null argument or negative count");
  std::vector<int32_t> nb;
  for (const auto &kv : t.duals) if (nb.empty() || nb.back() != kv.first.first) nb.push_back(kv.first.first);
  *n_out = (int32_t)nb.size();
  if ((int32_t)nb.size() > max_n) return pgo_fail(h, 2, std::string(what) + ": room for " + std::to_string(max_n) + " ids, " + std::to_string(nb.size()) + " needed");
  std::copy(nb.begin(), nb.end(), ids_out);
  return 0;
}

// the broadcast payload for one neighbour: its frame ids ascending, y_l [n][D] and (if not null) y_r [n][D]
template <int W>
static int arock_export(d2pgo_handle *h, const ArockTable<W> &t, const char *what, int D, int32_t neighbour, int32_t max_n, int32_t *n_out,
                        int64_t *frame_ids, double *local_out, double *remote_out) {
  if (!n_out || max_n < 0 || (max_n > 0 && (!frame_ids || !local_out))) return pgo_fail(h, 1, std::string(what) + ": null argument or negative count");
  auto lo = t.duals.lower_bound(std::make_pair(neighbour, INT64_MIN)), hi = t.duals.upper_bound(std::make_pair(neighbour, INT64_MAX));
  const int32_t cnt = (int32_t)std::distance(lo, hi);
  *n_out = cnt;
  if (cnt > max_n) return pgo_fail(h, 2, std::string(what) + ": room for " + std::to_string(max_n) + " duals, " + std::to_string(cnt) + " needed");
  int k = 0;
  for (auto it = lo; it != hi; ++it) frame_ids[k++] = it->first.second;
  arock_flatten(lo, hi, D, local_out, remote_out);
  return 0;
}

// the dual table, in table order, to the device: pose of each dual, the pose -> duals CSR, y_r, y_l, q_init
template <class H>
static int arock_sync(d2pgo_handle *h) {
  const auto &duals = h->pose_table.duals;
  const size_t N = h->ids.size(), K = duals.size(), D = H::D;
  std::vector<int> pose(K), ptr(N + 1, 0), of(K);
  std::vector<double> yr(K * D), yl(K * D), qi(N * 4, 0.0);
  size_t k = 0;
  for (const auto &kv : duals) { pose[k] = h->index.at(kv.first.second); ptr[pose[k] + 1]++; k++; }
  arock_flatten(duals.begin(), duals.end(), (int)D, yl.data(), yr.data());
  for (size_t i = 0; i < N; i++) ptr[i + 1] += ptr[i];
  { std::vector<int> fill(ptr.begin(), ptr.end() - 1);
    for (size_t j = 0; j < K; j++) of[fill[pose[j]]++] = (int)j; }
  if (H::arock_qinit) for (size_t i = 0; i < N; i++) memcpy(&qi[i * 4], h->qinit.at(h->ids[i]).data(), 32);
  PCK(h->d_ak_pose.alloc(K)); PCK(h->d_ak_of.alloc(K)); PCK(h->d_ak_ptr.alloc(N + 1)); PCK(h->d_ak_yr.alloc(K * D)); PCK(h->d_ak_yl.alloc(K * D));
  PCK(h->d_ak_qinit.alloc(N * 4)); PCK(h->d_ak_lin[0].alloc(K * (D + D * D))); PCK(h->d_ak_lin[1].alloc(K * (D + D * D)));
  if (K) {
    PCK(cudaMemcpyAsync(h->d_ak_pose.p, pose.data(), K * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_ak_of.p, of.data(), K * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_ak_yr.p, yr.data(), K * D * 8, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_ak_yl.p, yl.data(), K * D * 8, cudaMemcpyHostToDevice, h->stream));
  }
  PCK(cudaMemcpyAsync(h->d_ak_ptr.p, ptr.data(), (N + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(h->d_ak_qinit.p, qi.data(), N * 32, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  h->ak_n = (int)K;
  return pgo_alloc_cost_part(h);
}

// every pose needs an owner (and, 6-DoF, a q_init) before the table can be built
static int arock_check_poses(d2pgo_handle *h, const char *what) {
  if (!h->arock) return pgo_fail(h, 5, std::string(what) + ": the handle is not in ARock mode (d2pgo_arock_enable)");
  for (int64_t id : h->ids) {
    if (!h->owner.count(id)) return pgo_fail(h, 2, std::string(what) + ": pose id " + std::to_string(id) + " has no owner agent (d2pgo_arock_enable)");
    if (h->dof == 6 && !h->qinit.count(id)) return pgo_fail(h, 2, std::string(what) + ": pose id " + std::to_string(id) + " has no q_init (d2pgo_arock_enable)");
  }
  return 0;
}

extern "C" {

int d2pgo_default_arock_config(d2pgo_arock_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->self_id = 0; c->dual_state_init_to_zero = 0; c->rho_frame_T = 0.1; c->rho_frame_theta = 0.1; c->eta_k = 0.9;
  return 0;
}

int d2pgo_arock_enable(d2pgo_handle *h, const d2pgo_arock_config *cfg, int32_t n, const int64_t *ids, const int32_t *owner, const double *q_init4) {
  if (!h) return 1;
  if (!cfg || n < 0 || (n > 0 && (!ids || !owner))) return pgo_fail(h, 1, "arock_enable: null argument or negative count");
  if (h->comm) return pgo_fail(h, 5, "arock_enable: the handle has a communicator (edge sharding and ARock are different splits of the graph)");
  if (!(std::isfinite(cfg->rho_frame_T) && cfg->rho_frame_T >= 0.0 && std::isfinite(cfg->rho_frame_theta) && cfg->rho_frame_theta >= 0.0 && std::isfinite(cfg->eta_k)))
    return pgo_fail(h, 2, "arock_enable: rho_frame_T, rho_frame_theta must be finite and non-negative, eta_k finite");
  std::vector<std::array<double, 4>> q(n);
  for (int k = 0; k < n; k++) {
    auto it = h->index.find(ids[k]);
    if (it == h->index.end()) return pgo_fail(h, 2, "arock_enable: unknown pose id " + std::to_string(ids[k]));
    const double *src = q_init4 ? q_init4 + (size_t)k * 4 : h->chart ? &h->chart_qinit[(size_t)it->second * 4] : &h->poses[(size_t)it->second * 8 + 3];
    if (h->dof == 6 && !chart_unit(src, q[k].data()))
      return pgo_fail(h, 2, "arock_enable: pose id " + std::to_string(ids[k]) + ": non-finite or zero q_init");
  }
  h->arock = true; h->acfg = *cfg;
  for (int k = 0; k < n; k++) { h->owner[ids[k]] = owner[k]; if (h->dof == 6) h->qinit[ids[k]] = q[k]; }
  h->ak_n = -1;
  return 0;
}

int d2pgo_arock_receive(d2pgo_handle *h, int32_t sender, int32_t target, int32_t n, const int64_t *frame_ids, int32_t dim, const double *duals) {
  if (!h) return 1;
  if (!h->arock) return pgo_fail(h, 5, "arock_receive: the handle is not in ARock mode (d2pgo_arock_enable)");
  if (int rc = arock_receive_check(h, "arock_receive", h->dof, sender, n, frame_ids, dim, duals)) return rc;
  arock_queue(h->pose_table, sender, target, n, frame_ids, h->dof, duals);
  return 0;
}

int d2pgo_arock_step(d2pgo_handle *h, d2pgo_report *rep) {
  if (!h) return 1;
  if (h->ids.empty()) return pgo_fail(h, 1, "arock_step: no poses");
  if (int rc = arock_check_poses(h, "arock_step")) return rc;
  if (int rc = lm_refuse(h, "arock_step")) return rc;
  cudaSetDevice(h->cfg.device);
  return with_policy(h, [&](auto pol) -> int {   // one policy for the dual coordinates, the solve and the dual update
    using H = decltype(pol);
    int rc;
    if (!h->uploaded && (rc = pgo_upload(h))) return rc;
    const int D = H::D, self = h->acfg.self_id;
    const std::vector<char> in = arock_in_problem(h);
    auto &duals = h->pose_table.duals;
    // 1. receiveAll / processPGOData, on the live table
    arock_apply_inbox(h, h->pose_table, in, D, duals);
    h->pose_table.inbox.clear();
    // 2. scanAndCreateDualStates (ARock.cpp:192-208): a dual for every frame of another agent, from x(f) or zero.  The q_init
    // table goes to the device first (arock_sync) so that the coordinates can be taken there.
    if ((rc = arock_sync<H>(h))) return rc;
    std::vector<double> coord;
    if (!h->acfg.dual_state_init_to_zero && (rc = H::arock_coords(h, coord))) return rc;
    bool created = false;
    for (size_t i = 0; i < h->ids.size(); i++) {
      const int32_t o = h->owner.at(h->ids[i]);
      if (!in[i] || o == self) continue;
      const auto key = std::make_pair(o, h->ids[i]);
      if (duals.count(key)) continue;
      d2pgo_host::ArockDual<6> nd; memset(&nd, 0, sizeof nd);
      if (!h->acfg.dual_state_init_to_zero) { memcpy(nd.yl, &coord[i * D], D * 8); memcpy(nd.yr, &coord[i * D], D * 8); }
      duals.emplace(key, nd); created = true;
    }
    // 3. setDualStateFactors + solveLocalStep: the LM solve with the proximal terms towards y_r
    if (created && (rc = arock_sync<H>(h))) return rc;
    if ((rc = pgo_minimize<H>(h, rep, true))) return rc;
    // 4. updateDualStates at the solved poses, which pgo_solve leaves in buffer 0
    const PgoArockDev ak = pgo_arock_view(h, 0);
    if (ak.n_dual > 0) {
      H::arock_update(h->stream, h->d_x[0].p, ak);
      PCK(cudaGetLastError());
      std::vector<double> yl((size_t)ak.n_dual * D);
      PCK(cudaMemcpyAsync(yl.data(), h->d_ak_yl.p, yl.size() * 8, cudaMemcpyDeviceToHost, h->stream));
      PCK(cudaStreamSynchronize(h->stream));
      arock_set_yl(duals, D, yl.data());
    }
    return 0;
  });
}

int d2pgo_arock_neighbours(d2pgo_handle *h, int32_t max_n, int32_t *n_out, int32_t *ids_out) {
  if (!h) return 1;
  if (!h->arock) return pgo_fail(h, 5, "arock_neighbours: the handle is not in ARock mode (d2pgo_arock_enable)");
  return arock_neighbours(h, h->pose_table, "arock_neighbours", max_n, n_out, ids_out);
}

int d2pgo_arock_duals(d2pgo_handle *h, int32_t neighbour, int32_t max_n, int32_t *n_out, int64_t *frame_ids, double *local_out, double *remote_out) {
  if (!h) return 1;
  if (!h->arock) return pgo_fail(h, 5, "arock_duals: the handle is not in ARock mode (d2pgo_arock_enable)");
  return arock_export(h, h->pose_table, "arock_duals", h->dof, neighbour, max_n, n_out, frame_ids, local_out, remote_out);
}

int d2pgo_debug_arock_terms(d2pgo_handle *h, double *out, int64_t out_doubles) {
  if (!h) return 1;
  if (int rc = arock_check_poses(h, "debug_arock_terms")) return rc;
  const size_t K = h->pose_table.duals.size(), D = h->dof, W = D + D * D;
  if ((size_t)out_doubles < K * W) return pgo_fail(h, 2, "debug_arock_terms: buffer too small: " + std::to_string(K * W) + " doubles needed");
  if (!out && K) return pgo_fail(h, 1, "debug_arock_terms: null argument");
  if (!K) return 0;
  cudaSetDevice(h->cfg.device);
  int rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  if ((rc = with_policy(h, [h](auto pol) {
        using H = decltype(pol);
        if (int e = arock_sync<H>(h)) return e;
        H::lin_arock(h->stream, pgo_view(h, 0), pgo_arock_view(h, 0), h->d_cost_part.p);
        return 0;
      }))) return rc;
  PCK(cudaGetLastError());
  std::vector<double> tmp(K * W);
  PCK(cudaMemcpyAsync(tmp.data(), h->d_ak_lin[0].p, K * W * 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  for (size_t k = 0; k < K; k++) for (size_t q = 0; q < W; q++) out[k * W + q] = tmp[q * K + k];   // device layout is field-major
  return 0;
}

}  // extern "C"

// ---- sparse Cholesky (d2pgo_set_linear_solver) host side
template <class H>
static int pgo_exact_step(d2pgo_handle *h, double lambda, bool ark, double *out) {
  int rc;
  if ((rc = pgo_chol_prepare(h))) return rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  if (ark && (rc = arock_sync<H>(h))) return rc;
  double cost;
  if ((rc = pgo_linearize<H>(h, 0, 1, !h->gp_pose.empty(), ark, &cost))) return rc;
  bool failed = false;
  if ((rc = pgo_chol_step(h, 0, lambda, &failed))) return rc;
  PCK(cudaMemcpyAsync(out, h->d_dx.p, h->ids.size() * (size_t)H::D * 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  if (failed) { h->err = "debug_exact_step: the factorisation met a non-positive or non-finite pivot"; return 6; }
  return 0;
}

// the iterations of the last pgo_pcg and the relative residual sqrt(r.r / b.b) of its last update, read from the device (with
// max_it = 0 pgo_pcg reads nothing back): the r.r partials sit in the parity slot of the last iteration (cg_init: slot 1)
static int pcg_last_residual(d2pgo_handle *h, int32_t *iters, double *residual) {
  const PgoDev d = pgo_view(h, 0);
  PgoScalars s;
  PCK(cudaMemcpyAsync(&s, h->d_s.p, sizeof s, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  std::vector<double> part(d.nbp);
  const int slot = s.iters == 0 ? 1 : (s.iters - 1) & 1;
  PCK(cudaMemcpyAsync(part.data(), d.rr_part + (size_t)slot * d.nbp, (size_t)d.nbp * 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  double rr = 0.0;
  for (double v : part) rr += v;
  *iters = s.iters;
  *residual = s.bb > 0.0 ? std::sqrt(rr / s.bb) : 0.0;
  return 0;
}

// one PCG step of d2pgo_solve at the current poses (buffer 0), its iteration count and last relative residual
template <class H>
static int pgo_pcg_step(d2pgo_handle *h, double lambda, int max_it, double tol, bool ark, double *out, int32_t *iters, double *residual) {
  int rc;
  if (!h->uploaded && (rc = pgo_upload(h))) return rc;
  if (ark && (rc = arock_sync<H>(h))) return rc;
  const bool grav = !h->gp_pose.empty();
  double cost;
  if ((rc = pgo_linearize<H>(h, 0, 1, grav, ark, &cost))) return rc;
  PgoScalars s; memset(&s, 0, sizeof s);
  if ((rc = pgo_pcg<typename H::Kern>(h, 0, lambda, tol * tol, max_it, grav, ark, &s))) return rc;
  PCK(cudaMemcpyAsync(out, h->d_dx.p, h->ids.size() * (size_t)H::D * 8, cudaMemcpyDeviceToHost, h->stream));
  return pcg_last_residual(h, iters, residual);
}

extern "C" {

int d2pgo_set_linear_solver(d2pgo_handle *h, int32_t kind) {
  if (!h) return 1;
  if (kind != D2PGO_LINEAR_PCG && kind != D2PGO_LINEAR_SPARSE_CHOLESKY) {
    h->err = "set_linear_solver: unknown kind " + std::to_string(kind) + " (0 = PCG, 1 = sparse Cholesky)";
    return 2;
  }
  if (kind == D2PGO_LINEAR_SPARSE_CHOLESKY && h->comm) {
    h->err = "set_linear_solver: the handle has a communicator; the sparse Cholesky has no edge-sharded form";
    return 5;
  }
  if (kind == D2PGO_LINEAR_PCG && h->chol) {   // the factor's tables, fronts and graphs are not needed by PCG
    cudaSetDevice(h->cfg.device);
    cudaStreamSynchronize(h->stream);
    h->chol.reset();
  }
  h->linear_solver = kind;
  return 0;
}

int d2pgo_cholesky_stats(d2pgo_handle *h, d2pgo_cholesky_info *out) {
  if (!h || !out) return 1;
  memset(out, 0, sizeof *out);
  if (h->ids.empty()) return 0;
  if (int rc = pgo_chol_analyse(h)) return rc;   // analysis only: no device work
  d2pgo_chol::fill_info(h->chol->sym, out);
  out->factorizations = h->chol->factorizations; out->failed_factorizations = h->chol->failed;
  out->factor_ms = h->chol->factor_ms; out->solve_ms = h->chol->solve_ms;
  return 0;
}

int d2pgo_debug_exact_step(d2pgo_handle *h, double lambda, double *dx_out, int64_t out_doubles) {
  if (!h) return 1;
  if (!dx_out || h->ids.empty()) { h->err = "debug_exact_step: null argument or no poses"; return 1; }
  if ((size_t)out_doubles < h->ids.size() * (size_t)h->dof) { h->err = "debug_exact_step: buffer too small: " + std::to_string(h->ids.size() * h->dof) + " doubles needed"; return 2; }
  if (!(lambda >= 0.0 && std::isfinite(lambda))) { h->err = "debug_exact_step: lambda must be finite and non-negative"; return 2; }
  if (h->comm) { h->err = "debug_exact_step: the handle has a communicator"; return 5; }
  if (h->arock) if (int rc = arock_check_poses(h, "debug_exact_step")) return rc;
  cudaSetDevice(h->cfg.device);
  return with_policy(h, [&](auto pol) { return pgo_exact_step<decltype(pol)>(h, lambda, h->arock, dx_out); });
}

int d2pgo_debug_pcg_step(d2pgo_handle *h, double lambda, int32_t max_it, double tol, double *dx_out, int64_t out_doubles,
                         int32_t *iters_out, double *residual_out) {
  if (!h) return 1;
  if (!dx_out || !iters_out || !residual_out || h->ids.empty()) { h->err = "debug_pcg_step: null argument or no poses"; return 1; }
  if ((size_t)out_doubles < h->ids.size() * (size_t)h->dof) { h->err = "debug_pcg_step: buffer too small: " + std::to_string(h->ids.size() * h->dof) + " doubles needed"; return 2; }
  if (!(lambda >= 0.0 && std::isfinite(lambda)) || !(tol >= 0.0 && std::isfinite(tol)) || max_it < 0) {
    h->err = "debug_pcg_step: lambda and tol must be finite and non-negative, max_it non-negative";
    return 2;
  }
  if (h->comm) { h->err = "debug_pcg_step: the handle has a communicator"; return 5; }
  if (h->arock) if (int rc = arock_check_poses(h, "debug_pcg_step")) return rc;
  cudaSetDevice(h->cfg.device);
  return with_policy(h, [&](auto pol) { return pgo_pcg_step<decltype(pol)>(h, lambda, max_it, tol, h->arock, dx_out, iters_out, residual_out); });
}

int d2pgo_debug_cholesky_system(d2pgo_handle *h, double *diag_out, double *b_out, int32_t max_pairs, int32_t *n_pairs_out,
                                int32_t *pair_ab_out, double *pair_out) {
  if (!h) return 1;
  if (!diag_out || !b_out || !n_pairs_out || max_pairs < 0 || (max_pairs > 0 && (!pair_ab_out || !pair_out))) {
    h->err = "debug_cholesky_system: null argument or negative count";
    return 1;
  }
  const d2pgo_chol::Numeric *c = h->chol.get();
  if (!c || !c->has_system || c->sym.D != h->dof || c->sym.fixed != h->fixed || c->sym.ea != h->ea || c->sym.eb != h->eb) {
    h->err = "debug_cholesky_system: no sparse-Cholesky step on the handle's current structure";
    return 5;
  }
  *n_pairs_out = c->sym.n_pairs;
  if (max_pairs < c->sym.n_pairs) { h->err = "debug_cholesky_system: room for " + std::to_string(max_pairs) + " pairs, " + std::to_string(c->sym.n_pairs) + " needed"; return 2; }
  cudaSetDevice(h->cfg.device);
  return h->chol->system(h->stream, diag_out, b_out, max_pairs, pair_ab_out, pair_out, h->err);
}

}  // extern "C"

// ---- chordal rotation initialisation host side (d2pgo_rot_init)

// Eigen's toRotationMatrix polynomial (q2R of d2ba_math.cuh) on the host, row-major, of the normalised quaternion (Swarm::Pose
// normalises its attitude)
static void rot_quat_R(const double *q_xyzw, double *R) {
  const double n = std::sqrt(q_xyzw[0] * q_xyzw[0] + q_xyzw[1] * q_xyzw[1] + q_xyzw[2] * q_xyzw[2] + q_xyzw[3] * q_xyzw[3]);
  const double x = q_xyzw[0] / n, y = q_xyzw[1] / n, z = q_xyzw[2] / n, w = q_xyzw[3] / n;
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  const double m[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  for (int k = 0; k < 9; k++) R[k] = m[k];
}

static int rot_find(std::vector<int> &uf, int i) {
  while (uf[i] != i) { uf[i] = uf[uf[i]]; i = uf[i]; }
  return i;
}

// one row system on the inner handle h (poses and edges uploaded; errors are reported there): linearise at x = 0 rows, one
// undamped Gauss-Newton step by the block-Jacobi PCG of d2pgo_solve, x + dx into h->d_x[1]
static int rot_solve_row(d2pgo_handle *h, double tol2, int max_it, int *iters, double *residual) {
  typedef PgoRotRow P;
  int rc;
  const PgoDev d = pgo_view(h, 0);
  const PgoPriorDev pr = pgo_prior_view(h, 0);
  if (d.n_edge > 0) k_pgo_lin<P><<<(d.n_edge + 127) / 128, 128, 0, h->stream>>>(d, h->d_cost_part.p, 1);
  k_pgo_gD<P, false><<<d.nbp, 128, 0, h->stream>>>(d, h->d_g[0].p, h->d_D[0].p, pr);
  PgoScalars s; memset(&s, 0, sizeof s);
  if ((rc = pgo_pcg<P>(h, 0, 0.0, tol2, max_it, false, false, &s))) return rc;
  k_pgo_retract<P><<<d.nbp, 128, 0, h->stream>>>(d, h->d_x[1].p);
  return pcg_last_residual(h, iters, residual);
}

// the rotation initialisation problem both entry points solve: ego_of[i] = the entry of pose i in ego_ids (gravity rows only),
// -1 = none; the frames the edges name (all of them: the reference's all_frames, :444-450); the edges that give rows; the
// union-find of free frames joined by the edges with both ends free, and which of its components are anchored
struct RotProblem { std::vector<int> ego_of, uf, used; std::vector<char> named, anchored; int dropped = 0; };

// the checks of the settings both configs share, the ego attitudes and the edges; an edge from a fixed frame anchors its free
// end's component
static int rot_problem(d2pgo_handle *h, const char *what, const d2pgo_rot_init_config &cfg, int32_t n_ego, const int64_t *ego_ids,
                       const double *ego_poses7, RotProblem &s) {
  const std::string w(what);
  if (!(std::isfinite(cfg.pcg_tolerance) && cfg.pcg_tolerance >= 0.0) || cfg.pcg_max_iterations < 0 ||
      (cfg.enable_gravity_prior && !std::isfinite(cfg.gravity_sqrt_info)))
    return pgo_fail(h, 2, w + ": non-finite or negative pcg_tolerance, gravity_sqrt_info or pcg_max_iterations");
  const int N = (int)h->ids.size(), E = (int)h->ea.size();
  s.ego_of.assign(N, -1);
  for (int k = 0; k < n_ego; k++) {
    const std::string which = w + ": ego pose " + std::to_string(k) + " (id " + std::to_string(ego_ids[k]) + ")";
    auto it = h->index.find(ego_ids[k]);
    if (it == h->index.end()) return pgo_fail(h, 2, which + ": unknown pose id");
    if (s.ego_of[it->second] >= 0) return pgo_fail(h, 2, which + ": duplicate id");
    s.ego_of[it->second] = k;
    if (!all_finite(ego_poses7 + (size_t)k * 7, 7)) return pgo_fail(h, 2, which + ": non-finite value");
    const double *q = ego_poses7 + (size_t)k * 7 + 3;
    if (!(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0)) return pgo_fail(h, 2, which + ": zero quaternion");
  }
  s.named.assign(N, 0); s.uf.resize(N); s.used.clear(); s.dropped = 0;
  for (int i = 0; i < N; i++) s.uf[i] = i;
  for (int e = 0; e < E; e++) {
    const int a = h->ea[e], b = h->eb[e];
    s.named[a] = s.named[b] = 1;
    const bool fa = h->fixed[a] != 0, fb = h->fixed[b] != 0;
    if (a == b || fb) { s.dropped++; continue; }   // self loop, both fixed, or b fixed with a free (the :84 quirk)
    const double *q = &h->rel[(size_t)e * 8 + 3], *S = &h->sinfo[(size_t)e * 36];
    if (!all_finite(q, 4) || !(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0) || !all_finite(S, 36))
      return pgo_fail(h, 2, w + ": edge " + std::to_string(e) + ": non-finite or zero relative rotation or square-root information");
    if (fa && !all_finite(&h->poses[(size_t)a * 8 + 3], 4))
      return pgo_fail(h, 2, w + ": edge " + std::to_string(e) + ": non-finite attitude of its fixed frame");
    s.used.push_back(e);
    if (!fa) s.uf[rot_find(s.uf, a)] = rot_find(s.uf, b);
  }
  s.anchored.assign(N, 0);
  for (int e : s.used) if (h->fixed[h->ea[e]]) s.anchored[rot_find(s.uf, h->eb[e])] = 1;
  return 0;
}

// the free frames solved, ascending pose index: every free frame an edge names, refused if its attitude is not finite, its
// component is not anchored or, with gravity rows, it has no ego pose
static int rot_frames(d2pgo_handle *h, const char *what, RotProblem &s, bool grav, std::vector<int> &frames) {
  for (int i = 0; i < (int)h->ids.size(); i++) {
    if (!s.named[i] || h->fixed[i]) continue;
    const std::string fid = std::string(what) + ": frame id " + std::to_string(h->ids[i]);
    if (!all_finite(&h->poses[(size_t)i * 8 + 3], 4)) return pgo_fail(h, 2, fid + ": non-finite attitude");
    if (!s.anchored[rot_find(s.uf, i)]) return pgo_fail(h, 2, fid + ": its component of free frames is not anchored (A^T A is singular)");
    if (grav && s.ego_of[i] < 0) return pgo_fail(h, 2, fid + ": gravity rows are on and the frame has no ego pose");
    frames.push_back(i);
  }
  return 0;
}

// the inner handle of the row systems (dof 3, on h's stream) with the rows of the used edges: R_ab normalised, S = s I3 with
// s = |S[3:6, 3:6]|_F; Rfix[N][9] the rotations of the fixed frames those edges start from
static d2pgo_handle *rot_inner_edges(d2pgo_handle *h, const std::vector<int> &used, std::vector<double> &Rfix) {
  if (!h->rot) { h->rot.reset(new d2pgo_handle()); h->rot->dof = 3; }
  d2pgo_handle *r = h->rot.get();
  r->cfg = h->cfg; r->stream = h->stream;   // borrowed: r->own_stream stays false
  r->ea.clear(); r->eb.clear(); r->rel.clear(); r->sinfo.clear();
  for (int e : used) {
    r->ea.push_back(h->ea[e]); r->eb.push_back(h->eb[e]);
    const double *q = &h->rel[(size_t)e * 8 + 3], *S = &h->sinfo[(size_t)e * 36];
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double rel[8] = {0, 0, 0, q[0] / n, q[1] / n, q[2] / n, q[3] / n, 0};
    r->rel.insert(r->rel.end(), rel, rel + 8);
    double s2 = 0.0;   // |S[3:6, 3:6]|_F
    for (int i = 3; i < 6; i++) for (int j = 3; j < 6; j++) s2 += S[i * 6 + j] * S[i * 6 + j];
    const double s = std::sqrt(s2), Si[9] = {s, 0, 0, 0, s, 0, 0, 0, s};
    r->sinfo.insert(r->sinfo.end(), Si, Si + 9);
  }
  Rfix.assign(h->ids.size() * 9, 0.0);
  for (int e : used) if (h->fixed[h->ea[e]]) rot_quat_R(&h->poses[(size_t)h->ea[e] * 8 + 3], &Rfix[(size_t)h->ea[e] * 9]);
  return r;
}

// rows from the fixed virtual nodes base + j of r (its poses already sized) to the frames to[j], with R_ab = I, S = w I3
static void rot_unit_rows(d2pgo_handle *r, int base, const std::vector<int> &to, double w) {
  const double Si[9] = {w, 0, 0, 0, w, 0, 0, 0, w}, rel[8] = {0, 0, 0, 0, 0, 0, 1, 0};
  for (size_t j = 0; j < to.size(); j++) {
    r->ea.push_back(base + (int)j); r->eb.push_back(to[j]);
    r->rel.insert(r->rel.end(), rel, rel + 8); r->sinfo.insert(r->sinfo.end(), Si, Si + 9);
  }
}

// solveLinearRot (rotation_initialization_base.hpp:178-213): the three row systems on the inner handle.  Nodes: the handle's
// poses, then one fixed virtual node per dual prior, then (k = 2, gravity rows) one per solved frame.  Rows: the used edges;
// the dual priors, one to each frame of prior_pose with weight w, whose virtual node k_rotinit_arock_targets sets to row k of
// y_r of the dual d_prior[j] in d_yr; on k = 2 the gravity rows g (r_f^2 - R_ego^T e3), the virtual node holding R_ego^T e3.
// sol[k] = the solution of row system k ([nodes][8]); the per-row CG counts and residuals go to R.
static int rot_solve_rows(d2pgo_handle *h, const d2pgo_rot_init_config &cfg, const RotProblem &s, const std::vector<int> &frames,
                          const double *ego_poses7, const std::vector<int> &prior_pose, double w, const int *d_prior,
                          const double *d_yr, Buf<double> (&sol)[3], d2pgo_rot_init_report &R) {
  const int N = (int)h->ids.size(), P = (int)prior_pose.size();
  const bool grav = cfg.enable_gravity_prior != 0;
  std::vector<double> Rfix;
  d2pgo_handle *r = rot_inner_edges(h, s.used, Rfix);
  rot_unit_rows(r, N, prior_pose, w);
  const int Nn = N + P + (grav ? (int)frames.size() : 0);
  const double tol2 = cfg.pcg_tolerance * cfg.pcg_tolerance;
  for (int k = 0; k < 3; k++) {
    r->ids.assign(Nn, 0); r->fixed.assign(Nn, 1);
    for (int f : frames) r->fixed[f] = 0;
    r->poses.assign((size_t)Nn * 8, 0.0);
    for (int i = 0; i < N; i++) if (r->fixed[i]) for (int c = 0; c < 3; c++) r->poses[(size_t)i * 8 + c] = Rfix[(size_t)i * 9 + k * 3 + c];
    if (k == 2 && grav) {
      for (size_t j = 0; j < frames.size(); j++) {
        double Re[9];
        rot_quat_R(ego_poses7 + (size_t)s.ego_of[frames[j]] * 7 + 3, Re);
        for (int c = 0; c < 3; c++) r->poses[(N + P + j) * 8 + c] = Re[6 + c];   // R_ego^T e3 = third row of R_ego
      }
      rot_unit_rows(r, N + P, frames, cfg.gravity_sqrt_info);
    }
    int rc;
    if ((rc = pgo_upload(r))) return pgo_fail(h, rc, r->err);
    if (P) k_rotinit_arock_targets<<<(P + 127) / 128, 128, 0, h->stream>>>(P, k, d_prior, d_yr, r->d_x[0].p + (size_t)N * 8);
    if ((rc = rot_solve_row(r, tol2, cfg.pcg_max_iterations, &R.pcg_iterations[k], &R.residual[k]))) return pgo_fail(h, rc, r->err);
    PCK(sol[k].alloc((size_t)Nn * 8));
    PCK(cudaMemcpyAsync(sol[k].p, r->d_x[1].p, (size_t)Nn * 64, cudaMemcpyDeviceToDevice, h->stream));
  }
  return 0;
}

// the projection onto SO(3) of the F solved frames: project(fr, x, part, nb) launches the caller's kernel on the frame indices
// fr, the poses x ([N][8], from and back to poses) and nb per-block partials of the state changes; their mean over the frames
// goes to *state_changes
template <class Project>
static int rot_project(d2pgo_handle *h, const std::vector<int> &frames, std::vector<double> &poses, double *state_changes, Project project) {
  const int N = (int)h->ids.size(), F = (int)frames.size(), nb = (F + 127) / 128;
  Buf<double> x, part; Buf<int> fr;
  PCK(x.alloc((size_t)N * 8)); PCK(part.alloc(nb)); PCK(fr.alloc(F));
  PCK(cudaMemcpyAsync(x.p, poses.data(), (size_t)N * 64, cudaMemcpyHostToDevice, h->stream));
  PCK(cudaMemcpyAsync(fr.p, frames.data(), (size_t)F * 4, cudaMemcpyHostToDevice, h->stream));
  project(fr.p, x.p, part.p, nb);
  k_pgo_sum<<<1, 128, 0, h->stream>>>(part.p, nb, h->rot->d_cost.p);
  PCK(cudaGetLastError());
  double chg = 0.0;
  PCK(cudaMemcpyAsync(&chg, h->rot->d_cost.p, 8, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaMemcpyAsync(poses.data(), x.p, (size_t)N * 64, cudaMemcpyDeviceToHost, h->stream));
  PCK(cudaStreamSynchronize(h->stream));
  *state_changes = chg / F;
  return 0;
}

// the device time since h->ev0, once the stream has drained
static int rot_device_ms(d2pgo_handle *h, double *ms_out) {
  PCK(cudaEventRecord(h->ev1, h->stream));
  PCK(cudaEventSynchronize(h->ev1));
  float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  *ms_out = ms;
  return 0;
}

extern "C" {

int d2pgo_default_rot_init_config(d2pgo_rot_init_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->enable_gravity_prior = 0; c->pcg_max_iterations = 20000; c->gravity_sqrt_info = 10.0; c->pcg_tolerance = 1e-12;
  return 0;
}

static int rot_init_run(d2pgo_handle *h, const d2pgo_rot_init_config *cfg, int32_t n_ego, const int64_t *ego_ids, const double *ego_poses7,
                        d2pgo_rot_init_report *report) {
  if (!h) return 1;
  if (!cfg || n_ego < 0 || (n_ego > 0 && (!ego_ids || !ego_poses7))) return pgo_fail(h, 1, "rot_init: null argument or negative count");
  if (h->dof != 6) return pgo_fail(h, 5, "rot_init: the handle was created with pose_dof = 4; rotation initialisation acts on 6-DoF poses");
  if (h->comm) return pgo_fail(h, 5, "rot_init: a communicator is attached (edge-sharded rotation initialisation is not supported)");
  if (h->arock) return pgo_fail(h, 5, "rot_init: the handle is in ARock mode (d2pgo runs the distributed RotationInitARock there)");
  if (h->ids.empty()) return pgo_fail(h, 1, "rot_init: the handle has no poses");
  RotProblem s;
  std::vector<int> frames;
  int rc;
  if ((rc = rot_problem(h, "rot_init", *cfg, n_ego, ego_ids, ego_poses7, s))) return rc;
  if ((rc = rot_frames(h, "rot_init", s, cfg->enable_gravity_prior != 0, frames))) return rc;
  d2pgo_rot_init_report R; memset(&R, 0, sizeof R);
  R.frames = (int)frames.size(); R.edges_used = (int)s.used.size(); R.edges_dropped = s.dropped;
  std::vector<double> poses = h->poses;
  cudaSetDevice(h->cfg.device);
  auto device = [&]() -> int {
    PCK(cudaEventRecord(h->ev0, h->stream));
    if (!frames.empty()) {
      Buf<double> sol[3];
      if ((rc = rot_solve_rows(h, *cfg, s, frames, ego_poses7, {}, 0.0, nullptr, nullptr, sol, R))) return rc;
      auto project = [&](const int *fr, double *x, double *part, int nb) {
        k_rotinit_project<<<nb, 128, 0, h->stream>>>((int)frames.size(), fr, sol[0].p, sol[1].p, sol[2].p, x, part);
      };
      if ((rc = rot_project(h, frames, poses, &R.state_changes, project))) return rc;
    }
    return rot_device_ms(h, &R.device_ms);
  };
  if ((rc = device())) return pgo_fail(h, rc, "rot_init: " + h->err);
  h->poses.swap(poses);   // commit: the solved attitudes; the next d2pgo_solve uploads them
  h->uploaded = false;
  if (report) *report = R;
  return 0;
}

// on a chart handle the initialisation runs on the composed attitudes; each frame's q_init then becomes its attitude after it --
// the solved frames' the initialised one, every other frame's its current one (recoverRotationLLT, :360-389) --, and p and theta
// keep every bit
int d2pgo_rot_init(d2pgo_handle *h, const d2pgo_rot_init_config *cfg, int32_t n_ego, const int64_t *ego_ids, const double *ego_poses7,
                   d2pgo_rot_init_report *report) {
  if (!h || !h->chart) return rot_init_run(h, cfg, n_ego, ego_ids, ego_poses7, report);
  std::vector<double> state = chart_poses(h);
  state.swap(h->poses);
  const int rc = rot_init_run(h, cfg, n_ego, ego_ids, ego_poses7, report);
  if (!rc) for (size_t i = 0; i < h->ids.size(); i++) chart_unit(&h->poses[i * 8 + 3], &h->chart_qinit[i * 4]);
  h->poses.swap(state);
  h->uploaded = false;
  return rc;
}

}  // extern "C"

// ---- distributed rotation initialisation host side (d2pgo_arock_rot_*)

// w = |getSqrtInfoMatRot()|_F of a dual prior Swarm::PosePrior(f, Y_r, rho_rot_mat I3) (setDualStateFactors,
// rotation_initialization_arock.hpp:52-57).  ASSUMED: the 3x3 argument is information whose Cholesky factor is the square root
// sqrt(rho) I3, so w = sqrt(3 rho).
static double rot_dual_weight(double rho_rot_mat) { return std::sqrt(3.0 * rho_rot_mat); }

// what every d2pgo_arock_rot_* call needs: a 6-DoF handle in ARock mode; and a step or a receipt, one whose perturbation solve
// has not started
static int rot_arock_check(d2pgo_handle *h, const char *what, bool changes) {
  if (h->dof != 6) return pgo_fail(h, 5, std::string(what) + ": the handle was created with pose_dof = 4; rotation initialisation acts on 6-DoF poses");
  if (!h->arock) return pgo_fail(h, 5, std::string(what) + ": the handle is not in ARock mode (d2pgo_arock_enable)");
  if (changes && !h->pose_table.duals.empty()) return pgo_fail(h, 5, std::string(what) + ": the ARock pose dual table is not empty (rotation initialisation precedes the perturbation solve)");
  return 0;
}

extern "C" {

int d2pgo_default_arock_rot_init_config(d2pgo_arock_rot_init_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->enable_gravity_prior = 0; c->pcg_max_iterations = 20000; c->gravity_sqrt_info = 10.0; c->pcg_tolerance = 1e-12; c->rho_rot_mat = 0.1;
  return 0;
}

int d2pgo_arock_rot_receive(d2pgo_handle *h, int32_t sender, int32_t target, int32_t n, const int64_t *frame_ids, int32_t dim,
                            const double *duals, const double *poses7) {
  if (!h) return 1;
  int rc;
  if ((rc = rot_arock_check(h, "arock_rot_receive", true))) return rc;
  if (h->chart) return pgo_fail(h, 5, "arock_rot_receive: the handle is in the perturbation chart; the distributed rotation initialisation precedes it (d2pgo_set_chart after it takes its attitudes as q_init)");
  if (n > 0 && !poses7) return pgo_fail(h, 1, "arock_rot_receive: null argument or negative count");
  if ((rc = arock_receive_check(h, "arock_rot_receive", 9, sender, n, frame_ids, dim, duals))) return rc;
  if (!all_finite(poses7, (size_t)n * 7)) return pgo_fail(h, 2, "arock_rot_receive: non-finite pose");
  for (int k = 0; k < n; k++) {
    const double *q = poses7 + (size_t)k * 7 + 3;
    if (!(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] > 0.0)) return pgo_fail(h, 2, "arock_rot_receive: frame id " + std::to_string(frame_ids[k]) + ": zero quaternion");
  }
  // inputDPGOData (:216-235): the sender's frames take the sender's pose (position and attitude) and their attitude-init, now
  for (int k = 0; k < n; k++) {
    auto it = h->index.find(frame_ids[k]);
    if (it == h->index.end()) continue;
    auto o = h->owner.find(frame_ids[k]);
    if (o == h->owner.end() || o->second != sender) continue;
    const double *p = poses7 + (size_t)k * 7, *q = p + 3;
    memcpy(&h->poses[(size_t)it->second * 8], p, 56);
    const double s = 1.0 / std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    h->qinit[frame_ids[k]] = {q[0] * s, q[1] * s, q[2] * s, q[3] * s};
    h->uploaded = false;
  }
  arock_queue(h->rot_table, sender, target, n, frame_ids, 9, duals);
  return 0;
}

int d2pgo_arock_rot_init_step(d2pgo_handle *h, const d2pgo_arock_rot_init_config *cfg, int32_t n_ego, const int64_t *ego_ids,
                              const double *ego_poses7, d2pgo_rot_init_report *report) {
  if (!h) return 1;
  if (!cfg || n_ego < 0 || (n_ego > 0 && (!ego_ids || !ego_poses7))) return pgo_fail(h, 1, "arock_rot_init_step: null argument or negative count");
  int rc;
  if ((rc = rot_arock_check(h, "arock_rot_init_step", true))) return rc;
  if (h->chart) return pgo_fail(h, 5, "arock_rot_init_step: the handle is in the perturbation chart; the distributed rotation initialisation precedes it (d2pgo_set_chart after it takes its attitudes as q_init)");
  if (h->ids.empty()) return pgo_fail(h, 1, "arock_rot_init_step: the handle has no poses");
  if ((rc = arock_check_poses(h, "arock_rot_init_step"))) return rc;
  d2pgo_rot_init_config rcfg;   // the fields the two configs share
  rcfg.enable_gravity_prior = cfg->enable_gravity_prior; rcfg.pcg_max_iterations = cfg->pcg_max_iterations;
  rcfg.gravity_sqrt_info = cfg->gravity_sqrt_info; rcfg.pcg_tolerance = cfg->pcg_tolerance;
  RotProblem s;
  if ((rc = rot_problem(h, "arock_rot_init_step", rcfg, n_ego, ego_ids, ego_poses7, s))) return rc;
  if (!(std::isfinite(cfg->rho_rot_mat) && cfg->rho_rot_mat >= 0.0)) return pgo_fail(h, 2, "arock_rot_init_step: non-finite or negative rho_rot_mat");
  const int N = (int)h->ids.size(), self = h->acfg.self_id;
  // 1. receiveAll / processPGOData on a copy of the table, for the frames the problem estimates (an edge names them)
  auto duals = h->rot_table.duals;
  arock_apply_inbox(h, h->rot_table, s.named, 9, duals);
  // 3. scanAndCreateDualStates (:79-102): every edge end another agent owns gets the dual (owner, f), zero, if it has none
  for (size_t e = 0; e < h->ea.size(); e++)
    for (int i : {h->ea[e], h->eb[e]}) {
      const int32_t o = h->owner.at(h->ids[i]);
      if (o == self) continue;
      const auto key = std::make_pair(o, h->ids[i]);
      if (!duals.count(key)) { d2pgo_host::ArockDual<9> nd; memset(&nd, 0, sizeof nd); duals.emplace(key, nd); }
    }
  // 4. setDualStateFactors (:32-61): a prior per dual on a free frame; with the fixed-frame edge rows they anchor the components
  std::vector<int> dual_pose, prior_dual, prior_pose;
  for (const auto &kv : duals) {
    const int i = h->index.at(kv.first.second);
    if (!h->fixed[i]) { prior_dual.push_back((int)dual_pose.size()); prior_pose.push_back(i); s.anchored[rot_find(s.uf, i)] = 1; }
    dual_pose.push_back(i);
  }
  for (int i = 0; i < N; i++)
    if (s.named[i] && h->fixed[i] && !all_finite(&h->poses[(size_t)i * 8 + 3], 4))
      return pgo_fail(h, 2, "arock_rot_init_step: frame id " + std::to_string(h->ids[i]) + ": non-finite attitude");
  std::vector<int> frames;
  if ((rc = rot_frames(h, "arock_rot_init_step", s, rcfg.enable_gravity_prior != 0, frames))) return rc;
  std::vector<unsigned char> owned;
  for (int i : frames) owned.push_back(h->owner.at(h->ids[i]) == self);
  // R_state of every named frame: kept, or R(attitude) when the frame first enters a step (PGOState::addFrame)
  std::vector<double> rstate((size_t)N * 9, 0.0);
  for (int i = 0; i < N; i++) {
    auto it = h->rot_state.find(h->ids[i]);
    if (it != h->rot_state.end()) memcpy(&rstate[(size_t)i * 9], it->second.data(), 72);
    else if (s.named[i]) rot_quat_R(&h->poses[(size_t)i * 8 + 3], &rstate[(size_t)i * 9]);
  }
  const int K = (int)duals.size(), P = (int)prior_dual.size(), F = (int)frames.size();
  std::vector<double> yl((size_t)K * 9), yr((size_t)K * 9);
  arock_flatten(duals.begin(), duals.end(), 9, yl.data(), yr.data());
  d2pgo_rot_init_report R; memset(&R, 0, sizeof R);
  R.frames = F; R.edges_used = (int)s.used.size(); R.edges_dropped = s.dropped;
  std::vector<double> poses = h->poses;
  cudaSetDevice(h->cfg.device);
  auto device = [&]() -> int {
    PCK(cudaEventRecord(h->ev0, h->stream));
    // the dual table and the rotation states to the device
    PCK(h->d_rk_pose.alloc(K)); PCK(h->d_rk_prior.alloc(P)); PCK(h->d_rk_yl.alloc((size_t)K * 9)); PCK(h->d_rk_yr.alloc((size_t)K * 9));
    PCK(h->d_rk_state.alloc((size_t)N * 9));
    if (K) {
      PCK(cudaMemcpyAsync(h->d_rk_pose.p, dual_pose.data(), (size_t)K * 4, cudaMemcpyHostToDevice, h->stream));
      PCK(cudaMemcpyAsync(h->d_rk_yl.p, yl.data(), (size_t)K * 72, cudaMemcpyHostToDevice, h->stream));
      PCK(cudaMemcpyAsync(h->d_rk_yr.p, yr.data(), (size_t)K * 72, cudaMemcpyHostToDevice, h->stream));
    }
    if (P) PCK(cudaMemcpyAsync(h->d_rk_prior.p, prior_dual.data(), (size_t)P * 4, cudaMemcpyHostToDevice, h->stream));
    PCK(cudaMemcpyAsync(h->d_rk_state.p, rstate.data(), (size_t)N * 72, cudaMemcpyHostToDevice, h->stream));
    if (F) {
      // 5. solveLinearRot, with the dual priors
      Buf<double> sol[3];
      if ((rc = rot_solve_rows(h, rcfg, s, frames, ego_poses7, prior_pose, rot_dual_weight(cfg->rho_rot_mat), h->d_rk_prior.p, h->d_rk_yr.p, sol, R))) return rc;
      // 6. recoverRotationLLT: R_state = M, the owned frames' attitudes; state_changes = the mean over the free frames
      Buf<unsigned char> own;
      PCK(own.alloc(F));
      PCK(cudaMemcpyAsync(own.p, owned.data(), (size_t)F, cudaMemcpyHostToDevice, h->stream));
      auto project = [&](const int *fr, double *x, double *part, int nb) {
        k_rotinit_arock_project<<<nb, 128, 0, h->stream>>>(F, fr, own.p, sol[0].p, sol[1].p, sol[2].p, h->d_rk_state.p, x, part);
      };
      if ((rc = rot_project(h, frames, poses, &R.state_changes, project))) return rc;
    }
    // 7. updateDualStates on every dual, at R_state
    if (K) k_rotinit_arock_update<<<(K + 127) / 128, 128, 0, h->stream>>>(K, h->d_rk_pose.p, h->d_rk_state.p, h->d_rk_yr.p, h->d_rk_yl.p, h->acfg.eta_k);
    PCK(cudaGetLastError());
    if (K) PCK(cudaMemcpyAsync(yl.data(), h->d_rk_yl.p, (size_t)K * 72, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaMemcpyAsync(rstate.data(), h->d_rk_state.p, (size_t)N * 72, cudaMemcpyDeviceToHost, h->stream));
    return rot_device_ms(h, &R.device_ms);
  };
  if ((rc = device())) return pgo_fail(h, rc, "arock_rot_init_step: " + h->err);
  // commit: the table, the states of the named frames, the owned frames' attitudes and their q_init (so that the first
  // d2pgo_arock_step starts from theta = 0 at them); the inbox has been processed
  arock_set_yl(duals, 9, yl.data());
  h->rot_table.duals.swap(duals);
  h->rot_table.inbox.clear();
  for (int i = 0; i < N; i++) if (s.named[i]) memcpy(h->rot_state[h->ids[i]].data(), &rstate[(size_t)i * 9], 72);
  for (size_t j = 0; j < frames.size(); j++) {
    if (!owned[j]) continue;
    const double *q = &poses[(size_t)frames[j] * 8 + 3];
    const double n = 1.0 / std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    h->qinit[h->ids[frames[j]]] = {q[0] * n, q[1] * n, q[2] * n, q[3] * n};
  }
  h->poses.swap(poses);
  h->uploaded = false; h->ak_n = -1;
  if (report) *report = R;
  return 0;
}

int d2pgo_arock_rot_neighbours(d2pgo_handle *h, int32_t max_n, int32_t *n_out, int32_t *ids_out) {
  if (!h) return 1;
  if (int rc = rot_arock_check(h, "arock_rot_neighbours", false)) return rc;
  return arock_neighbours(h, h->rot_table, "arock_rot_neighbours", max_n, n_out, ids_out);
}

int d2pgo_arock_rot_duals(d2pgo_handle *h, int32_t neighbour, int32_t max_n, int32_t *n_out, int64_t *frame_ids, double *local9,
                          double *remote9, double *poses7) {
  if (!h) return 1;
  int rc;
  if ((rc = rot_arock_check(h, "arock_rot_duals", false))) return rc;
  if ((rc = arock_export(h, h->rot_table, "arock_rot_duals", 9, neighbour, max_n, n_out, frame_ids, local9, remote9))) return rc;
  if (poses7) for (int k = 0; k < *n_out; k++) memcpy(poses7 + (size_t)k * 7, &h->poses[(size_t)h->index.at(frame_ids[k]) * 8], 56);
  return 0;
}

int d2pgo_debug_arock_rot_state(d2pgo_handle *h, double *state9_out, uint8_t *flag_out, int32_t max_duals, int32_t *n_duals_out,
                                int32_t *neighbour_out, int64_t *frame_out, double *local9_out, double *remote9_out) {
  if (!h) return 1;
  if (int rc = rot_arock_check(h, "debug_arock_rot_state", false)) return rc;
  if (!state9_out || !flag_out || !n_duals_out || max_duals < 0 ||
      (max_duals > 0 && (!neighbour_out || !frame_out || !local9_out || !remote9_out))) return pgo_fail(h, 1, "debug_arock_rot_state: null argument or negative count");
  const size_t N = h->ids.size();
  std::vector<char> named(N, 0);
  for (size_t e = 0; e < h->ea.size(); e++) named[h->ea[e]] = named[h->eb[e]] = 1;
  for (size_t i = 0; i < N; i++) {
    auto it = h->rot_state.find(h->ids[i]);
    for (int c = 0; c < 9; c++) state9_out[i * 9 + c] = it == h->rot_state.end() ? 0.0 : it->second[c];
    flag_out[i] = !named[i] ? 0 : h->fixed[i] ? 2 : 1;
  }
  const auto &duals = h->rot_table.duals;
  const int32_t K = (int32_t)duals.size();
  *n_duals_out = K;
  if (K > max_duals) return pgo_fail(h, 2, "debug_arock_rot_state: room for " + std::to_string(max_duals) + " duals, " + std::to_string(K) + " needed");
  int k = 0;
  for (const auto &kv : duals) { neighbour_out[k] = kv.first.first; frame_out[k] = kv.first.second; k++; }
  arock_flatten(duals.begin(), duals.end(), 9, local9_out, remote9_out);
  return 0;
}

}  // extern "C"

// ---- minimiser selection and its reports (include/d2pgo.h d2pgo_set_minimizer)
extern "C" {

int d2pgo_default_ceres_lm_config(d2pgo_ceres_lm_config *c) {
  if (!c) return 1;
  memset(c, 0, sizeof *c);
  c->max_num_iterations = 50; c->max_num_consecutive_invalid_steps = 5; c->jacobi_scaling = 1;
  c->max_solver_time_in_seconds = 0.0; c->initial_trust_region_radius = 1e4; c->max_trust_region_radius = 1e16;
  c->min_trust_region_radius = 1e-32; c->min_relative_decrease = 1e-3; c->min_lm_diagonal = 1e-6; c->max_lm_diagonal = 1e32;
  c->function_tolerance = 1e-6; c->gradient_tolerance = 1e-10; c->parameter_tolerance = 1e-8;
  return 0;
}

int d2pgo_set_minimizer(d2pgo_handle *h, int32_t kind, const d2pgo_ceres_lm_config *cfg) {
  if (!h) return 1;
  if (kind == D2PGO_MINIMIZER_RESTATED) { h->minimizer = kind; return 0; }
  if (kind != D2PGO_MINIMIZER_CERES_LM)
    return pgo_fail(h, 2, "set_minimizer: unknown kind " + std::to_string(kind) + " (0 = the restated LM loop, 1 = ceres LM)");
  d2pgo_ceres_lm_config c;
  if (cfg) c = *cfg; else d2pgo_default_ceres_lm_config(&c);
  const double v[10] = {c.max_solver_time_in_seconds, c.initial_trust_region_radius, c.max_trust_region_radius, c.min_trust_region_radius,
                        c.min_relative_decrease, c.min_lm_diagonal, c.max_lm_diagonal, c.function_tolerance, c.gradient_tolerance, c.parameter_tolerance};
  for (double x : v)
    if (!(std::isfinite(x) && x >= 0.0)) return pgo_fail(h, 2, "set_minimizer: every real field must be finite and non-negative");
  if (c.max_num_iterations < 0 || c.max_num_consecutive_invalid_steps < 0 || (c.jacobi_scaling != 0 && c.jacobi_scaling != 1))
    return pgo_fail(h, 2, "set_minimizer: max_num_iterations and max_num_consecutive_invalid_steps must be >= 0, jacobi_scaling 0 or 1");
  if (!(c.min_trust_region_radius > 0.0 && c.min_trust_region_radius <= c.initial_trust_region_radius &&
        c.initial_trust_region_radius <= c.max_trust_region_radius))
    return pgo_fail(h, 2, "set_minimizer: need 0 < min_trust_region_radius <= initial_trust_region_radius <= max_trust_region_radius");
  if (!(c.min_lm_diagonal > 0.0 && c.min_lm_diagonal <= c.max_lm_diagonal))
    return pgo_fail(h, 2, "set_minimizer: need 0 < min_lm_diagonal <= max_lm_diagonal");
  h->minimizer = kind; h->lm_cfg = c;
  return 0;
}

int d2pgo_minimizer_report(d2pgo_handle *h, d2pgo_minimizer_summary *out) {
  if (!h || !out) return 1;
  if (!h->lm_ran) return pgo_fail(h, 5, "minimizer_report: the last solve or ARock step did not run the ceres minimiser");
  *out = h->lm_report;
  return 0;
}

int d2pgo_debug_minimizer_trace(d2pgo_handle *h, int32_t max, int32_t *n_out, d2pgo_minimizer_iteration *out) {
  if (!h || !n_out || (max > 0 && !out)) return 1;
  if (!h->lm_ran) return pgo_fail(h, 5, "debug_minimizer_trace: the last solve or ARock step did not run the ceres minimiser");
  *n_out = h->lm_trace_n;
  if (max < h->lm_trace_n) return pgo_fail(h, 2, "debug_minimizer_trace: " + std::to_string(h->lm_trace_n) + " records, room for " + std::to_string(max));
  cudaSetDevice(h->cfg.device);
  if (h->lm_trace_n > 0) {
    PCK(cudaMemcpyAsync(out, h->d_lm_trace.p, (size_t)h->lm_trace_n * sizeof *out, cudaMemcpyDeviceToHost, h->stream));
    PCK(cudaStreamSynchronize(h->stream));
  }
  return 0;
}

}  // extern "C"

// ---- the perturbation chart's entry points (include/d2pgo.h d2pgo_set_chart)
extern "C" {

int d2pgo_set_chart(d2pgo_handle *h, int32_t chart, int32_t n, const int64_t *ids, const double *q_init4) {
  if (!h) return 1;
  if (chart != D2PGO_CHART_RETRACTION && chart != D2PGO_CHART_PERTURB)
    return pgo_fail(h, 2, "set_chart: unknown chart " + std::to_string(chart) + " (0 = retraction, 1 = perturbation)");
  if (h->dof != 6) return pgo_fail(h, 5, "set_chart: the handle was created with pose_dof = 4; d2pgo builds RelPoseFactor4D there in either mode");
  if (h->comm) return pgo_fail(h, 5, "set_chart: the handle has a communicator; the perturbation chart has no edge-sharded form");
  if (h->arock && !h->pose_table.duals.empty())
    return pgo_fail(h, 5, "set_chart: the handle's ARock duals are held in the other chart's coordinates (enter the chart before the first d2pgo_arock_step)");
  if (n < 0 || (n > 0 && !ids)) return pgo_fail(h, 1, "set_chart: null argument or negative count");
  for (int k = 0; k < n; k++)
    if (!h->index.count(ids[k])) return pgo_fail(h, 2, "set_chart: unknown pose id " + std::to_string(ids[k]));
  // the attitudes as they stand, then every validation before anything changes
  std::vector<double> cur = h->chart ? chart_poses(h) : h->poses;
  const size_t N = h->ids.size();
  std::vector<double> qi(N * 4);
  for (size_t i = 0; i < N; i++)
    if (!chart_unit(&cur[i * 8 + 3], &qi[i * 4])) return pgo_fail(h, 2, "set_chart: pose id " + std::to_string(h->ids[i]) + ": non-finite or zero attitude");
  if (chart == D2PGO_CHART_PERTURB && q_init4)
    for (int k = 0; k < n; k++) {
      auto it = h->index.find(ids[k]);
      if (!chart_unit(q_init4 + (size_t)k * 4, &qi[(size_t)it->second * 4]))
        return pgo_fail(h, 2, "set_chart: pose id " + std::to_string(ids[k]) + ": non-finite or zero q_init");
    }
  if (chart == D2PGO_CHART_PERTURB) {   // PGOState::addFrame: x = [p, 0]
    for (size_t i = 0; i < N; i++) for (int k = 3; k < 8; k++) cur[i * 8 + k] = 0.0;
    h->chart_qinit.swap(qi);
  } else {
    h->chart_qinit.clear();
  }
  h->poses.swap(cur);
  h->chart = chart;
  h->uploaded = false;
  return 0;
}

int d2pgo_set_perturb(d2pgo_handle *h, int32_t n, const int64_t *ids, const double *x6) {
  if (!h) return 1;
  if (!h->chart) return pgo_fail(h, 5, "set_perturb: the handle is not in the perturbation chart (d2pgo_set_chart)");
  if (n < 0 || (n > 0 && (!ids || !x6))) return pgo_fail(h, 1, "set_perturb: null argument or negative count");
  std::vector<int> idx(n);
  for (int k = 0; k < n; k++) {
    auto it = h->index.find(ids[k]);
    if (it == h->index.end()) return pgo_fail(h, 2, "set_perturb: unknown pose id " + std::to_string(ids[k]));
    if (!all_finite(x6 + (size_t)k * 6, 6)) return pgo_fail(h, 2, "set_perturb: pose id " + std::to_string(ids[k]) + ": non-finite value");
    idx[k] = it->second;
  }
  for (int k = 0; k < n; k++) memcpy(&h->poses[(size_t)idx[k] * 8], x6 + (size_t)k * 6, 48);
  if (n > 0) h->uploaded = false;
  return 0;
}

int d2pgo_get_perturb(d2pgo_handle *h, int32_t n, const int64_t *ids, double *x6_out, double *q_init4_out) {
  if (!h) return 1;
  if (!h->chart) return pgo_fail(h, 5, "get_perturb: the handle is not in the perturbation chart (d2pgo_set_chart)");
  if (n < 0 || (n > 0 && (!ids || !x6_out))) return pgo_fail(h, 1, "get_perturb: null argument or negative count");
  for (int k = 0; k < n; k++) {
    auto it = h->index.find(ids[k]);
    if (it == h->index.end()) return pgo_fail(h, 2, "get_perturb: unknown pose id " + std::to_string(ids[k]));
    memcpy(x6_out + (size_t)k * 6, &h->poses[(size_t)it->second * 8], 48);
    if (q_init4_out) memcpy(q_init4_out + (size_t)k * 4, &h->chart_qinit[(size_t)it->second * 4], 32);
  }
  return 0;
}

}  // extern "C"
