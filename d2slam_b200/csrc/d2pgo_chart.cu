// d2pgo_chart.cu -- the pose graph's perturbation chart (d2pgo_set_chart, include/d2pgo.h; d2pgo_chart.cuh): d2pgo's 6-DoF
// perturb_mode factors evaluated as the reference writes them, with their Jacobians in [p, theta], and the chart's retraction.
// A file of its own, so that d2pgo.o keeps exactly the kernels it had.
#include <math.h>

#include <cmath>

#include "d2ba_math.cuh"
#include "d2pgo_chart.cuh"

namespace d2pgo_chart {
using namespace d2ba;
namespace {

// ---- the perturbation chart (d2pgo_set_chart, d2pgo's perturb_mode): the state of a pose is the Euclidean 6-vector
// x = [p, theta] (POSE_PERTURB_6D), its attitude q = q_init (x) quatfromRotationVector(theta), and the factors are
// RelPoseFactorPerturbAD (RelPoseFactor.hpp:138-195) and GravityPriorPerturbAD (GravityPrior.hpp:8-46) evaluated as written:
// inside |theta| < 1e-2 the unnormalised [theta / 2, 1], the conjugate (not the inverse) of a non-unit q_a applied through
// Eigen's _transformVector, and Eigen's toRotationMatrix polynomial, which assumes a unit q.  Jacobians are with respect to
// [p, theta], as ceres' dual numbers give them.  Quaternions are [x y z w]; 4x4 matrices act on that order.

// quatfromRotationVector (utils.hpp:39-55) and dq [4][3] = d q / d theta
D2BA_DEV Q4 chart_dq(const double *th, double *dq) {
  const double n = sqrt(th[0] * th[0] + th[1] * th[1] + th[2] * th[2]);
  if (n < 1e-2) {   // deltaQ: [theta / 2, 1]
    for (int k = 0; k < 12; k++) dq[k] = k < 9 && k % 4 == 0 ? 0.5 : 0.0;
    return Q4{th[0] / 2.0, th[1] / 2.0, th[2] / 2.0, 1.0};
  }
  const double h = n / 2.0, s = sin(h), c = cos(h), u[3] = {th[0] / n, th[1] / n, th[2] / n};
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) dq[i * 3 + j] = s / n * ((i == j ? 1.0 : 0.0) - u[i] * u[j]) + 0.5 * c * u[i] * u[j];
    dq[9 + i] = -0.5 * s * u[i];
  }
  return Q4{u[0] * s, u[1] * s, u[2] * s, c};
}

// q (x) p = L(q) p and p (x) q = R(q) p, Hamilton products as Eigen forms them
D2BA_DEV void chart_qL(const Q4 &q, double *L) {
  const double m[16] = {q.w, -q.z, q.y, q.x, q.z, q.w, -q.x, q.y, -q.y, q.x, q.w, q.z, -q.x, -q.y, -q.z, q.w};
  for (int k = 0; k < 16; k++) L[k] = m[k];
}
D2BA_DEV void chart_qR(const Q4 &q, double *R) {
  const double m[16] = {q.w, q.z, -q.y, q.x, -q.z, q.w, q.x, q.y, q.y, -q.x, q.w, q.z, -q.x, -q.y, -q.z, q.w};
  for (int k = 0; k < 16; k++) R[k] = m[k];
}

// q = q_init (x) dq(theta) of the state x6 = [p, theta] and Jq [4][3] = d q / d theta
D2BA_DEV Q4 chart_att(const double *x6, const double *qi, double *Jq) {
  double dqt[12], L[16];
  const Q4 q0 = qload(qi), dq = chart_dq(x6 + 3, dqt);
  chart_qL(q0, L);
  for (int i = 0; i < 4; i++) for (int j = 0; j < 3; j++) {
    double t = 0.0;
    for (int k = 0; k < 4; k++) t += L[i * 4 + k] * dqt[k * 3 + j];
    Jq[i * 3 + j] = t;
  }
  return qmul(q0, dq);
}

// RelPoseFactorPerturbAD at x_a = [p_a, theta_a], x_b: with q_c = q_a.conjugate() = (v, w), t = p_b - p_a,
//   p_ab = t + w (2 v x t) + v x (2 v x t)   (Eigen's _transformVector),  dq = q_meas (x) (q_c (x) q_b).conjugate(),
//   r = S [p_ab - p_meas ; 2 vec(dq)]
D2BA_DEV void chart_edge_eval(const double *xa, const double *xb, const double *qia, const double *qib, const double *rel, const double *S,
                              double *r, double *J0, double *J1) {
  double Ja[12], Jb[12];
  const Q4 qa = chart_att(xa, qia, Ja), qb = chart_att(xb, qib, Jb), qm = qload(rel + 3);
  const Q4 qc = Q4{-qa.x, -qa.y, -qa.z, qa.w};
  const double t[3] = {xb[0] - xa[0], xb[1] - xa[1], xb[2] - xa[2]};
  const double v[3] = {qc.x, qc.y, qc.z}, w = qc.w;
  const double uv[3] = {2.0 * (v[1] * t[2] - v[2] * t[1]), 2.0 * (v[2] * t[0] - v[0] * t[2]), 2.0 * (v[0] * t[1] - v[1] * t[0])};
  const double vu[3] = {v[1] * uv[2] - v[2] * uv[1], v[2] * uv[0] - v[0] * uv[2], v[0] * uv[1] - v[1] * uv[0]};
  const double pab[3] = {t[0] + w * uv[0] + vu[0], t[1] + w * uv[1] + vu[1], t[2] + w * uv[2] + vu[2]};
  const Q4 qab = qmul(qc, qb);
  const Q4 dq = qmul(qm, Q4{-qab.x, -qab.y, -qab.z, qab.w});
  const double raw[6] = {pab[0] - rel[0], pab[1] - rel[1], pab[2] - rel[2], 2.0 * dq.x, 2.0 * dq.y, 2.0 * dq.z};
  for (int i = 0; i < 6; i++) { double s = 0; for (int k = 0; k < 6; k++) s += S[i * 6 + k] * raw[k]; r[i] = s; }
  if (!J0) return;
  // d p_ab / d t = M = I + 2 w [v]x + 2 [v]x^2,  d p_ab / d v = -2 w [t]x - [uv]x - 2 [v]x [t]x,  d p_ab / d w = uv
  const double Vx[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0}, Tx[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
  const double Ux[9] = {0, -uv[2], uv[1], uv[2], 0, -uv[0], -uv[1], uv[0], 0};
  double M[9], Pq[12];   // Pq [3][4]: d p_ab / d q_a (x y z w of q_a; q_c's vector part is minus q_a's)
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    double vv = 0.0, vt = 0.0;
    for (int k = 0; k < 3; k++) { vv += Vx[i * 3 + k] * Vx[k * 3 + j]; vt += Vx[i * 3 + k] * Tx[k * 3 + j]; }
    M[i * 3 + j] = (i == j ? 1.0 : 0.0) + 2.0 * w * Vx[i * 3 + j] + 2.0 * vv;
    Pq[i * 4 + j] = -(-2.0 * w * Tx[i * 3 + j] - Ux[i * 3 + j] - 2.0 * vt);
  }
  for (int i = 0; i < 3; i++) Pq[i * 4 + 3] = uv[i];
  // dq = L(q_m) C R(q_b) C q_a = L(q_m) C L(q_c) q_b, C = diag(-1, -1, -1, 1)
  double Lm[16], Rb[16], Lc[16], Da[12], Db[12];   // Da, Db [3][4]: d vec(dq) / d q_a, d q_b
  chart_qL(qm, Lm); chart_qR(qb, Rb); chart_qL(qc, Lc);
  for (int i = 0; i < 3; i++) for (int j = 0; j < 4; j++) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < 4; k++) {
      const double lk = Lm[i * 4 + k] * (k < 3 ? -1.0 : 1.0);
      a += lk * Rb[k * 4 + j] * (j < 3 ? -1.0 : 1.0);
      b += lk * Lc[k * 4 + j];
    }
    Da[i * 4 + j] = a; Db[i * 4 + j] = b;
  }
  double A0[36], A1[36];
  for (int k = 0; k < 36; k++) { A0[k] = 0.0; A1[k] = 0.0; }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    A0[i * 6 + j] = -M[i * 3 + j]; A1[i * 6 + j] = M[i * 3 + j];
    double pa = 0.0, ra = 0.0, rb = 0.0;
    for (int k = 0; k < 4; k++) { pa += Pq[i * 4 + k] * Ja[k * 3 + j]; ra += Da[i * 4 + k] * Ja[k * 3 + j]; rb += Db[i * 4 + k] * Jb[k * 3 + j]; }
    A0[i * 6 + 3 + j] = pa; A0[(3 + i) * 6 + 3 + j] = 2.0 * ra; A1[(3 + i) * 6 + 3 + j] = 2.0 * rb;
  }
  for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
    double t0 = 0, t1 = 0;
    for (int k = 0; k < 6; k++) { t0 += S[i * 6 + k] * A0[k * 6 + j]; t1 += S[i * 6 + k] * A1[k * 6 + j]; }
    J0[i * 6 + j] = t0; J1[i * 6 + j] = t1;
  }
}

// GravityPriorPerturbAD at x = [p, theta]: u = row 2 of toRotationMatrix(q) = [2 (xz - yw), 2 (yz + xw), 1 - 2 (x^2 + y^2)] by
// Eigen's polynomial, r = S^T (u - u_ego); J = d r / d theta (3x3 row-major; the position columns are zero)
D2BA_DEV void chart_gravity_eval(const double *x6, const double *qi, const double *ue, const double *S, double *r, double *J) {
  double Jq[12], R[9];
  const Q4 q = chart_att(x6, qi, Jq);
  q2R(q, R);
  const double du[3] = {R[6] - ue[0], R[7] - ue[1], R[8] - ue[2]};
  for (int i = 0; i < 3; i++) r[i] = S[i] * du[0] + S[3 + i] * du[1] + S[6 + i] * du[2];
  const double U[12] = {2 * q.z, -2 * q.w, 2 * q.x, -2 * q.y, 2 * q.w, 2 * q.z, 2 * q.y, 2 * q.x, -4 * q.x, -4 * q.y, 0.0, 0.0};   // d u / d q
  double G[9];
  for (int a = 0; a < 3; a++) for (int j = 0; j < 3; j++) { double t = 0.0; for (int k = 0; k < 4; k++) t += U[a * 4 + k] * Jq[k * 3 + j]; G[a * 3 + j] = t; }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) J[i * 3 + j] = S[i] * G[j] + S[3 + i] * G[3 + j] + S[6 + i] * G[6 + j];
}

__global__ void __launch_bounds__(128) k_chart_edges(int n_edge, const int *ea, const int *eb, const double *x, const double *qinit,
                                                      const double *rel, const double *sinfo, double *lin, double *cost_part, int want_jac) {
  constexpr int D = 6, DD = 36;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (e < n_edge) {
    const int a = ea[e], b = eb[e];
    double r[D], J0[DD], J1[DD];
    chart_edge_eval(x + (size_t)a * 8, x + (size_t)b * 8, qinit + (size_t)a * 4, qinit + (size_t)b * 4, rel + (size_t)e * 8,
                    sinfo + (size_t)e * DD, r, want_jac ? J0 : nullptr, J1);
    for (int k = 0; k < D; k++) c += 0.5 * r[k] * r[k];
    if (want_jac) {
      double *o = lin + e;   // field-major [D + 2 D^2][E], as k_pgo_lin writes it
      const size_t E = (size_t)n_edge;
      for (int k = 0; k < D; k++) o[k * E] = r[k];
      for (int k = 0; k < DD; k++) { o[(D + k) * E] = J0[k]; o[(D + DD + k) * E] = J1[k]; }
    }
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}

__global__ void __launch_bounds__(128) k_chart_priors(int n_prior, const int *pose, const double *u, const double *S, const double *x,
                                                       const double *qinit, double *lin, double *cost_part, int want_jac) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (k < n_prior) {
    const size_t i = (size_t)pose[k];
    double r[3], J[9];
    chart_gravity_eval(x + i * 8, qinit + i * 4, u + (size_t)k * 3, S + (size_t)k * 9, r, J);
    for (int a = 0; a < 3; a++) c += 0.5 * r[a] * r[a];
    if (want_jac) {
      double *o = lin + k;   // field-major [12][G], as k_pgo_prior_lin writes it
      const size_t G = (size_t)n_prior;
      for (int a = 0; a < 3; a++) o[a * G] = r[a];
      for (int a = 0; a < 9; a++) o[(3 + a) * G] = J[a];
    }
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}

__global__ void k_chart_retract(int n, const double *x, const unsigned char *fixed, const double *dx, double *x_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < 6; k++) x_out[(size_t)i * 8 + k] = fixed[i] ? x[(size_t)i * 8 + k] : x[(size_t)i * 8 + k] + dx[(size_t)i * 6 + k];
  x_out[(size_t)i * 8 + 6] = 0.0; x_out[(size_t)i * 8 + 7] = 0.0;
}

// ARock's proximal NormalPrior in the chart (ARock.cpp:284-291): the dual coordinates are the state itself, so per dual k on pose
// i, r = diag(wT I3, wR I3) (x_i - y_r) and the constant J = diag(wT I3, wR I3); records [6 + 36][K] field-major
__global__ void __launch_bounds__(128) k_chart_arock_lin(int n_dual, const int *pose, const double *x, const double *yr, double wT, double wR,
                                                          double *lin, double *cost_part) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  __shared__ double red[40];
  double c = 0.0;
  if (k < n_dual) {
    const double *xi = x + (size_t)pose[k] * 8, *y = yr + (size_t)k * 6;
    double *o = lin + k;
    const size_t K = (size_t)n_dual;
    for (int q = 0; q < 6; q++) {
      const double r = (q < 3 ? wT : wR) * (xi[q] - y[q]);
      c += 0.5 * r * r;
      o[q * K] = r;
    }
    for (int q = 0; q < 36; q++) o[(6 + q) * K] = q % 7 ? 0.0 : (q < 18 ? wT : wR);
  }
  c = block_sum(c, red);
  if (threadIdx.x == 0) cost_part[blockIdx.x] = c;
}

// updateDualStates (ARock.cpp:50-81) on the state: y_l -= eta ((y_l + y_r) / 2 - x_i), in the reference's order and rounding
__global__ void k_chart_arock_update(int n_dual, const int *pose, const double *x, const double *yr, double *yl, double eta) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_dual) return;
  const double *xi = x + (size_t)pose[k] * 8;
  for (int q = 0; q < 6; q++) {
    const double l = yl[(size_t)k * 6 + q];
    const double avg = __ddiv_rn(__dadd_rn(l, yr[(size_t)k * 6 + q]), 2.0);
    yl[(size_t)k * 6 + q] = __dsub_rn(l, __dmul_rn(__dsub_rn(avg, xi[q]), eta));
  }
}

}  // namespace

void arock_lin(cudaStream_t st, int n_dual, const int *pose, const double *x, const double *yr, double wT, double wR, double *lin,
               double *cost_part) {
  k_chart_arock_lin<<<(n_dual + 127) / 128, 128, 0, st>>>(n_dual, pose, x, yr, wT, wR, lin, cost_part);
}

void arock_update(cudaStream_t st, int n_dual, const int *pose, const double *x, const double *yr, double *yl, double eta) {
  k_chart_arock_update<<<(n_dual + 127) / 128, 128, 0, st>>>(n_dual, pose, x, yr, yl, eta);
}

void edges(cudaStream_t st, int n_edge, const int *ea, const int *eb, const double *x, const double *qinit, const double *rel,
           const double *sinfo, double *lin, double *cost_part, int want_jac) {
  k_chart_edges<<<(n_edge + 127) / 128, 128, 0, st>>>(n_edge, ea, eb, x, qinit, rel, sinfo, lin, cost_part, want_jac);
}

void priors(cudaStream_t st, int n_prior, const int *pose, const double *u, const double *S, const double *x, const double *qinit,
            double *lin, double *cost_part, int want_jac) {
  k_chart_priors<<<(n_prior + 127) / 128, 128, 0, st>>>(n_prior, pose, u, S, x, qinit, lin, cost_part, want_jac);
}

void retract(cudaStream_t st, int n_pose, const double *x, const unsigned char *fixed, const double *dx, double *x_out) {
  k_chart_retract<<<(n_pose + 127) / 128, 128, 0, st>>>(n_pose, x, fixed, dx, x_out);
}

}  // namespace d2pgo_chart
