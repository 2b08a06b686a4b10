// d2ba_kernels.cu -- sm_90a kernels of the sliding-window BA solver (DESIGN.md section 4).
//
//   k_state_prep      rotation matrices of every six-dof block
//   k_imu_prep        IMU sqrt-information U = chol(cov^-1)^T            (imu_factor.h:29)
//   k_prior_prep      A' = J_lin^T J_lin of the marginalisation prior
//   k_misc_lin        IMU + prior + ADMM terms -> Hcc, gc, cost          (one CTA / window)
//   k_proj_lin<..>    fused reprojection residual + Jacobian + Huber + DMMA J^T J accumulation
//   k_lm_gather       per-landmark reduction -> scaled coupling rows Wt, h, g
//   k_schur           S = Hcc + mu D^2 - Wt^T Wt  (fp64 tensor-core SYRK) + bordered rhs row
//   k_chol            blocked bordered Cholesky + back substitution        (one CTA / window)
//   k_step            landmark back-substitution, Cauchy point, dogleg, retraction
//   k_control         accept / reject, radius, convergence
//   k_cons_*          ADMM consensus pack / apply
#include <cuda_runtime.h>
#include <cstdio>
#include <stdint.h>
#include <map>
#include <mutex>
#include <type_traits>

#include "../../include/d2ba.h"
#include "d2ba_math.cuh"
#include "d2ba_proj.cuh"
#include "d2ba_types.cuh"

namespace d2ba {

// ------------------------------------------------------------------------------------------------
__global__ void k_state_prep(Dev d, int n6_total, int buf) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n6_total) return;
  const double *x = d.x6[buf] + (size_t)i * 8;
  q2R(qload(x + 3), d.R6[buf] + (size_t)i * 12);
}

// ------------------------------------------------------------------------------------------------
// sqrt_info = LLT(cov^-1).matrixL().transpose(): one thread per IMU factor (setup, once per finalize)
__global__ void k_imu_prep(Dev d, int n_imu) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_imu) return;
  const double *cov = d.imu_c + (size_t)f * kImuStride + 17 + 225;
  double *U = d.imu_U + (size_t)f * 225;
  double L[225], inv[225];
  for (int i = 0; i < 225; i++) L[i] = cov[i];
  // cholesky (lower) of cov
  for (int j = 0; j < 15; j++) {
    double dd = L[j * 15 + j];
    for (int k = 0; k < j; k++) dd -= L[j * 15 + k] * L[j * 15 + k];
    dd = sqrt(dd);
    L[j * 15 + j] = dd;
    for (int i = j + 1; i < 15; i++) {
      double s = L[i * 15 + j];
      for (int k = 0; k < j; k++) s -= L[i * 15 + k] * L[j * 15 + k];
      L[i * 15 + j] = s / dd;
    }
  }
  // inverse via two triangular solves per unit vector
  for (int c = 0; c < 15; c++) {
    double y[15], x[15];
    for (int i = 0; i < 15; i++) {
      double s = (i == c) ? 1.0 : 0.0;
      for (int k = 0; k < i; k++) s -= L[i * 15 + k] * y[k];
      y[i] = s / L[i * 15 + i];
    }
    for (int i = 14; i >= 0; i--) {
      double s = y[i];
      for (int k = i + 1; k < 15; k++) s -= L[k * 15 + i] * x[k];
      x[i] = s / L[i * 15 + i];
    }
    for (int i = 0; i < 15; i++) inv[i * 15 + c] = x[i];
  }
  for (int i = 0; i < 15; i++)
    for (int j = i + 1; j < 15; j++) { double m = 0.5 * (inv[i * 15 + j] + inv[j * 15 + i]); inv[i * 15 + j] = m; inv[j * 15 + i] = m; }
  for (int j = 0; j < 15; j++) {
    double dd = inv[j * 15 + j];
    for (int k = 0; k < j; k++) dd -= inv[j * 15 + k] * inv[j * 15 + k];
    dd = sqrt(dd);
    inv[j * 15 + j] = dd;
    for (int i = j + 1; i < 15; i++) {
      double s = inv[i * 15 + j];
      for (int k = 0; k < j; k++) s -= inv[i * 15 + k] * inv[j * 15 + k];
      inv[i * 15 + j] = s / dd;
    }
  }
  for (int i = 0; i < 15; i++)
    for (int j = 0; j < 15; j++) U[i * 15 + j] = (j >= i) ? inv[j * 15 + i] : 0.0;
}

// A' = J^T J of each window's prior (constant across iterations: the prior is linear in dx)
__global__ void k_prior_prep(Dev d) {
  const WinDesc &w = d.win[blockIdx.x];
  int m = w.prior_m;
  if (m <= 0) return;
  const double *J = d.prior_J + w.off_prior_J;
  double *A = d.prior_A + w.off_prior_J;
  for (int e = threadIdx.x; e < m * m; e += blockDim.x) {
    int i = e / m, j = e % m;
    double s = 0;
    for (int k = 0; k < m; k++) s += J[(size_t)k * m + i] * J[(size_t)k * m + j];
    A[e] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// IMU raw residual (15) and raw Jacobian (15 x 30: pose_i 6 | sb_i 9 | pose_j 6 | sb_j 9) before the
// sqrt-information is applied.  Same terms as IMUFactor::Evaluate (d2vins/src/factors/imu_factor.h:41-213)
// and IntegrationBase::evaluate (d2common/include/d2common/integration_base.h:201-227).
__device__ void imu_raw(const double *c, const double *pi, const double *si, const double *pj, const double *sj,
                        double g, double *res, double *J /*15x30 zeroed*/) {
  const double dt = c[0];
  const double *dp = c + 1, *dq = c + 4, *dv = c + 8, *ba0 = c + 11, *bg0 = c + 14, *Jp = c + 17;
  Q4 Qi = qload(pi + 3), Qj = qload(pj + 3), Dq = qload(dq);
  double Ri[9];
  q2R(Qi, Ri);
  auto jb = [&](int r, int col, double *o) {
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b = 0; b < 3; b++) o[a * 3 + b] = Jp[(r + a) * 15 + col + b];
  };
  double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
  jb(0, 9, dp_dba); jb(0, 12, dp_dbg); jb(3, 12, dq_dbg); jb(6, 9, dv_dba); jb(6, 12, dv_dbg);
  double dba[3] = {si[3] - ba0[0], si[4] - ba0[1], si[5] - ba0[2]};
  double dbg[3] = {si[6] - bg0[0], si[7] - bg0[1], si[8] - bg0[2]};
  double th[3], t1[3], t2[3];
  mv3(dq_dbg, dbg, th);
  Q4 cq = qmul(Dq, Q4{0.5 * th[0], 0.5 * th[1], 0.5 * th[2], 1.0});
  double cv[3], cp[3];
  mv3(dv_dba, dba, t1); mv3(dv_dbg, dbg, t2);
  for (int k = 0; k < 3; k++) cv[k] = dv[k] + t1[k] + t2[k];
  mv3(dp_dba, dba, t1); mv3(dp_dbg, dbg, t2);
  for (int k = 0; k < 3; k++) cp[k] = dp[k] + t1[k] + t2[k];
  double G[3] = {0, 0, g};
  double a1[3], a2[3], ra1[3], ra2[3];
  for (int k = 0; k < 3; k++) { a1[k] = 0.5 * G[k] * dt * dt + pj[k] - pi[k] - si[k] * dt; a2[k] = G[k] * dt + sj[k] - si[k]; }
  mtv3(Ri, a1, ra1); mtv3(Ri, a2, ra2);
  Q4 qij = qmul(qinv(Qi), Qj);
  Q4 er = qmul(qinv(cq), qij);
  for (int k = 0; k < 3; k++) { res[k] = ra1[k] - cp[k]; res[6 + k] = ra2[k] - cv[k]; res[9 + k] = sj[3 + k] - si[3 + k]; res[12 + k] = sj[6 + k] - si[6 + k]; }
  res[3] = 2 * er.x; res[4] = 2 * er.y; res[5] = 2 * er.z;
  if (!J) return;
  auto put = [&](int r, int col, const double *m, double s) {
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b = 0; b < 3; b++) J[(r + a) * 30 + col + b] = s * m[a * 3 + b];
  };
  auto skewm = [&](const double *v, double *o) { o[0] = 0; o[1] = -v[2]; o[2] = v[1]; o[3] = v[2]; o[4] = 0; o[5] = -v[0]; o[6] = -v[1]; o[7] = v[0]; o[8] = 0; };
  // bottom-right 3x3 of Qleft(a) (and of Qleft(a) Qright(b)), both after positify (utils.hpp:85-104)
  auto qleft3 = [&](Q4 a, double *o) {
    a = qpos(a);
    o[0] = a.w; o[1] = -a.z; o[2] = a.y; o[3] = a.z; o[4] = a.w; o[5] = -a.x; o[6] = -a.y; o[7] = a.x; o[8] = a.w;
  };
  double RiT[9] = {Ri[0], Ri[3], Ri[6], Ri[1], Ri[4], Ri[7], Ri[2], Ri[5], Ri[8]};
  double S[9], M[9], I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  // pose_i (cols 0..5)
  put(0, 0, RiT, -1.0);
  skewm(ra1, S); put(0, 3, S, 1.0);
  {
    Q4 a = qpos(qmul(qinv(Qj), Qi)), b = qpos(cq);
    double L3[9], R3[9];
    qleft3(a, L3);
    R3[0] = b.w; R3[1] = b.z; R3[2] = -b.y; R3[3] = -b.z; R3[4] = b.w; R3[5] = b.x; R3[6] = b.y; R3[7] = -b.x; R3[8] = b.w;
    mm3(L3, R3, M);
    double av[3] = {a.x, a.y, a.z}, bv[3] = {b.x, b.y, b.z};
    for (int r = 0; r < 3; r++) for (int cc = 0; cc < 3; cc++) M[r * 3 + cc] -= av[r] * bv[cc];
    put(3, 3, M, -1.0);
  }
  skewm(ra2, S); put(6, 3, S, 1.0);
  // sb_i (cols 6..14): V 6, BA 9, BG 12
  put(0, 6, RiT, -dt); put(0, 9, dp_dba, -1.0); put(0, 12, dp_dbg, -1.0);
  {
    double L3[9];
    qleft3(qmul(qmul(qinv(Qj), Qi), Dq), L3);  // uncorrected delta_q (imu_factor.h:159)
    mm3(L3, dq_dbg, M);
    put(3, 12, M, -1.0);
  }
  put(6, 6, RiT, -1.0); put(6, 9, dv_dba, -1.0); put(6, 12, dv_dbg, -1.0);
  put(9, 9, I3, -1.0); put(12, 12, I3, -1.0);
  // pose_j (cols 15..20)
  put(0, 15, RiT, 1.0);
  {
    double L3[9];
    qleft3(qmul(qmul(qinv(cq), qinv(Qi)), Qj), L3);
    put(3, 18, L3, 1.0);
  }
  // sb_j (cols 21..29)
  put(6, 21, RiT, 1.0); put(9, 24, I3, 1.0); put(12, 27, I3, 1.0);
}

D2BA_DEV void prior_dx_pose(const double *x, const double *x0, double *dx) {  // prior_factor.cpp:57-68
  dx[0] = x[0] - x0[0]; dx[1] = x[1] - x0[1]; dx[2] = x[2] - x0[2];
  Q4 e = qmul(qinv(qload(x0 + 3)), qload(x + 3));
  Q4 p = qpos(e);
  double s = (e.w >= 0) ? 2.0 : -2.0;  // the `!(w >= 0)` branch negates the positified vector again
  if (!(e.w >= 0)) { dx[3] = -2.0 * p.x; dx[4] = -2.0 * p.y; dx[5] = -2.0 * p.z; (void)s; }
  else { dx[3] = 2.0 * p.x; dx[4] = 2.0 * p.y; dx[5] = 2.0 * p.z; }
}

// ConsenusPoseFactor::Evaluate (consenus_factor.cpp:19-51): r = [wT (Rz^T (t - t_z) + t~) ; wq (2 vec(q_z^-1 q) + th~)],
// dT/dp = wT Rz^T, dth/dtheta = wq Qleft(q_z^-1 q)_3 (after positify).  NB the constructor's swap: wq = rho_T, wT = rho_theta.
D2BA_DEV void cons_eval(const double *x, const double *z, const double *tl, double wq, double wT, double *r, double *Rz, double *L3) {
  double dd[3] = {x[0] - z[0], x[1] - z[1], x[2] - z[2]}, t[3];
  Q4 qz = qload(z + 3);
  q2R(qz, Rz);
  mtv3(Rz, dd, t);
  Q4 qe = qmul(qinv(qz), qload(x + 3));
  r[0] = wT * (t[0] + tl[0]); r[1] = wT * (t[1] + tl[1]); r[2] = wT * (t[2] + tl[2]);
  r[3] = wq * (2 * qe.x + tl[3]); r[4] = wq * (2 * qe.y + tl[4]); r[5] = wq * (2 * qe.z + tl[5]);
  Q4 p = qpos(qe);
  L3[0] = p.w; L3[1] = -p.z; L3[2] = p.y; L3[3] = p.z; L3[4] = p.w; L3[5] = -p.x; L3[6] = -p.y; L3[7] = p.x; L3[8] = p.w;
}

// One CTA per window: zero Hcc/gc of the evaluated buffer, then add IMU, prior and ADMM terms.
// Runs before k_proj_lin (which adds the reprojection blocks with atomics).
constexpr int kMiscThreads = 256;
constexpr int kMiscImuChunk = 12;
__global__ void __launch_bounds__(kMiscThreads, 4) k_misc_lin(Dev d, int eval_cur) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || (!eval_cur && !ctl->step_valid)) return;
  const int buf = eval_cur ? ctl->cur : 1 - ctl->cur;
  const int tid = threadIdx.x, nt = blockDim.x;
  extern __shared__ double sm[];
  double *red = sm;             // 40
  double *Jr = sm + 40;         // prior scratch: dx, r, column map
  const int n = w.n_c, ld = w.ldh;
  double *H = d.Hcc[buf] + w.offH;
  double *g = d.gc[buf] + w.offc;
  const double *x6 = d.x6[buf] + (size_t)w.off6 * 8;
  const double *xsb = d.xsb[buf] + (size_t)w.offsb * 9;
  const double *xlm = d.xlm[buf] + w.offlm;
  const int *col6 = d.col6 + w.off6;
  const int *colsb = d.colsb + w.offsb;
#ifdef D2BA_MISC_TIMING
  long long mk[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; long long mq = clock64();
#define MLAP(k) do { __syncthreads(); long long t_ = clock64(); mk[k] += t_ - mq; mq = t_; } while (0)
#else
#define MLAP(k) do { } while (0)
#endif
  // ---- zero + IMU factors.  The raw residual / Jacobian of a factor is one long dependent chain (one lane per
  //      factor, all in warp 0); the other warps zero H / g and stage the sqrt-information meanwhile.  U J and
  //      [J r]^T [J r] then run on the fp64 tensor cores (m8n8k4), 8x8 output tiles spread over the warps.
  double cost = 0.0;
  // zero only the runs of Hcc some factor writes (lower triangle; the rest stays at the zero of the finalize-time memset)
  auto zero_H = [&](int t0, int tn) {
    const HSeg *sg = d.hseg + w.off_hseg;
    for (int e = t0; e < w.n_hseg; e += tn) {
      const HSeg q = sg[e];
      double *p = H + (size_t)q.row * ld + q.c0;
      for (int k = 0; k < q.len; k++) p[k] = 0.0;
    }
    for (int e = t0; e < n; e += tn) g[e] = 0.0;
  };
  zero_H(tid, nt);
  __syncthreads();
  // ---- prior: r = e0 + J dx ; H += J^T J ; g += J^T r
  if (w.prior_m > 0) {
    const int m = w.prior_m;
    double *dx = Jr, *r = Jr + m;
    int *cmap = reinterpret_cast<int *>(Jr + 2 * m);
    const PriorBlk *pb = d.prior_blk + w.off_prior_blk;
    if (tid < w.prior_nblk) {
      const PriorBlk &b = pb[tid];
      int col;
      if (b.kind == 0 || b.kind == 1) { prior_dx_pose(x6 + b.index * 8, b.x0, dx + b.off); col = col6[b.index]; }
      else if (b.kind == 2) { for (int q = 0; q < 9; q++) dx[b.off + q] = xsb[b.index * 9 + q] - b.x0[q]; col = colsb[b.index]; }
      else if (b.kind == 3) { dx[b.off] = d.xtd[buf][wi] - b.x0[0]; col = w.td_col; }
      else { dx[b.off] = xlm[b.index] - b.x0[0]; col = -1; }
      for (int q = 0; q < b.eff; q++) cmap[b.off + q] = col < 0 ? -1 : col + q;
    }
    __syncthreads();
    const double *J = d.prior_J + w.off_prior_J, *e0 = d.prior_e0 + w.off_prior_v, *A = d.prior_A + w.off_prior_J;
    {
      int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
      for (int i = warp; i < m; i += nw) {
        double s = 0;
        for (int j = lane; j < m; j += 32) s += J[(size_t)i * m + j] * dx[j];
        s = warp_sum(s);
        if (lane == 0) r[i] = e0[i] + s;
      }
    }
    __syncthreads();
    for (int j = tid; j < m; j += nt) {
      cost += 0.5 * r[j] * r[j];
      int gj = cmap[j];
      if (gj < 0) continue;
      double s = 0;
      for (int i = 0; i < m; i++) s += J[(size_t)i * m + j] * r[i];
      atomicAdd(&g[gj], s);
    }
    for (int e = tid; e < m * m; e += nt) {
      int i = e / m, j = e % m;
      int gi = cmap[i], gj = cmap[j];
      if (gi < 0 || gj < 0 || gj > gi) continue;   // lower triangle
      double v = A[e];
      if (v != 0.0) atomicAdd(&H[(size_t)gi * ld + gj], v);
    }
    __syncthreads();
  }
  MLAP(5);
  // ---- ADMM terms (ConsensusSolver::updateTilde, ConsensusSolver.cpp:108-164)
  if (w.admm_on) {
    const int *slot = d.slot6 + w.off6;
    for (int b = tid; b < w.n6; b += nt) {
      if (slot[b] < 0) continue;
      // ConsenusPoseFactor::Evaluate (consenus_factor.cpp:19-51); NB q weight = rho_T, T weight = rho_theta
      const double *z = d.z6 + (size_t)(w.off6 + b) * 8, *tl = d.tilde6 + (size_t)(w.off6 + b) * 6;
      const double *x = x6 + b * 8;
      const double wq = d.prm.rho_T, wT = d.prm.rho_theta;
      double Rz[9], L3[9], r[6];
      cons_eval(x, z, tl, wq, wT, r, Rz, L3);
      for (int q = 0; q < 6; q++) cost += 0.5 * r[q] * r[q];
      int c = col6[b];
      if (c < 0) continue;
      // J_T = wT Rz^T (3x3), J_q = wq L3
      for (int i = 0; i < 3; i++) {
        double gi = 0, gq = 0;
        for (int k = 0; k < 3; k++) { gi += wT * Rz[i * 3 + k] * r[k]; gq += wq * L3[k * 3 + i] * r[3 + k]; }
        atomicAdd(&g[c + i], gi); atomicAdd(&g[c + 3 + i], gq);
        for (int j = 0; j <= i; j++) {   // lower triangle
          double hT = 0, hq = 0;
          for (int k = 0; k < 3; k++) { hT += Rz[i * 3 + k] * Rz[j * 3 + k]; hq += L3[k * 3 + i] * L3[k * 3 + j]; }
          atomicAdd(&H[(size_t)(c + i) * ld + c + j], wT * wT * hT);
          atomicAdd(&H[(size_t)(c + 3 + i) * ld + c + 3 + j], wq * wq * hq);
        }
      }
    }
    // ceres::NormalPrior(A, x_ref): A = I for SPEED_BIAS / TD, rho_landmark for LANDMARK (:113-125)
    for (int e = tid; e < w.nsb * 9; e += nt) {
      int b = e / 9, q = e % 9;
      double rr = xsb[e] - d.sb_ref[(size_t)w.offsb * 9 + e];
      cost += 0.5 * rr * rr;
      int c = colsb[b];
      if (c >= 0) { atomicAdd(&H[(size_t)(c + q) * ld + c + q], 1.0); atomicAdd(&g[c + q], rr); }
    }
    if (tid == 0 && w.has_td) {
      double rr = d.xtd[buf][wi] - d.td_ref[wi];
      cost += 0.5 * rr * rr;
      if (w.td_col >= 0) { atomicAdd(&H[(size_t)w.td_col * ld + w.td_col], 1.0); atomicAdd(&g[w.td_col], rr); }
    }
    const double rl = d.prm.rho_landmark;
    for (int l = tid; l < w.nl; l += nt) {
      double rr = rl * (xlm[l] - d.lm_ref[w.offlm + l]);
      cost += 0.5 * rr * rr;
    }
  }
  cost = block_sum(cost, red);
  if (tid == 0) { ctl->cand_cost_misc = cost; }
#ifdef D2BA_MISC_TIMING
  MLAP(6);
  if (wi == 0 && tid == 0) printf("misc timing: zero %lld uload %lld imu_raw %lld UJ %lld JtJ %lld prior %lld tail %lld\n", mk[0], mk[1], mk[2], mk[3], mk[4], mk[5], mk[6]);
#endif
}

// ------------------------------------------------------------------------------------------------
// IMU factors: one WARP per factor over the whole batch (a window has only ~10 of them, so one CTA per window left the
// SMs mostly idle during the long dependent chain of the raw residual / Jacobian).  Lane 0 evaluates the raw terms
// (imu_raw), the warp then forms U [J r] and [J r]^T [J r] on the fp64 tensor cores (m8n8k4) and adds the lower triangle
// into Hcc / gc with L2 reductions.  Runs after k_misc_lin (which zeroed the written runs of Hcc) and adds its cost to it.
// k_imu_raw: one THREAD per factor -- the raw residual / Jacobian is one long dependent instruction stream, identical for every
// factor, so 32 factors run it in lockstep per warp (one warp per factor would issue the same stream 32 times).  Output to
// a global scratch [factor][465] whose never-written entries stay at the zero of the finalize-time memset.
__global__ void __launch_bounds__(32) k_imu_raw(Dev d, int eval_cur, int n_imu_total) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_imu_total) return;
  const ImuDesc im = d.imu[f];
  const WinDesc &w = d.win[im.win];
  const Ctl *ctl = d.ctl + im.win;
  if (ctl->done || (!eval_cur && !ctl->step_valid)) return;
  const int buf = eval_cur ? ctl->cur : 1 - ctl->cur;
  const double *x6 = d.x6[buf] + (size_t)w.off6 * 8, *xsb = d.xsb[buf] + (size_t)w.offsb * 9;
  double *raw = d.imu_raw + (size_t)f * (15 * 30 + 15);
  imu_raw(d.imu_c + (size_t)f * kImuStride, x6 + im.pi * 8, xsb + im.si * 9, x6 + im.pj * 8, xsb + im.sj * 9, d.prm.gravity, raw + 450, raw);
}
constexpr int kImuWarps = 4;
constexpr int kImuF = 15 * 30 + 15;   // doubles per factor for (J, r)
constexpr int kImuWarpDoubles = 2 * kImuF + 225 + 1;   // raw, U [J r], sqrt-information
__global__ void __launch_bounds__(kImuWarps * 32) k_imu_lin(Dev d, int eval_cur, int n_imu_total) {
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kImuWarps + warp;
  if (f >= n_imu_total) return;
  const ImuDesc im = d.imu[f];
  const int wi = im.win;
  const WinDesc &w = d.win[wi];
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || (!eval_cur && !ctl->step_valid)) return;
  const int buf = eval_cur ? ctl->cur : 1 - ctl->cur;
  double *raw = sm + (size_t)warp * kImuWarpDoubles, *fin = raw + kImuF, *Us = fin + kImuF;
  const int ld = w.ldh;
  double *H = d.Hcc[buf] + w.offH, *g = d.gc[buf] + w.offc;
  const int *col6 = d.col6 + w.off6, *colsb = d.colsb + w.offsb;
  // raw (J, r) of k_imu_raw and the sqrt-information: coalesced, all in flight
  {
    const double *Ug = d.imu_U + (size_t)f * 225, *rg = d.imu_raw + (size_t)f * kImuF;
    for (int e = lane; e < 225; e += 32) cp_async8(Us + e, Ug + e);
    for (int e = lane; e < kImuF; e += 32) cp_async8(raw + e, rg + e);
    cp_async_wait_all();
  }
  const int cols[4] = {col6[im.pi], colsb[im.si], col6[im.pj], colsb[im.sj]};
  const double *U = Us;
  __syncwarp();
  const int g4 = lane >> 2, q4 = lane & 3;
  // fin = U [Jraw | rraw]: 2 x 4 output tiles, K = 15 (4 k-steps, the 16th masked)
  for (int job = 0; job < 8; job++) {
    const int ti = job >> 2, tj = job & 3;
    const int i = 8 * ti + g4, bc = 8 * tj + g4;
    double c0 = 0.0, c1 = 0.0, av[4], bv[4];
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      const int kq = 4 * kk + q4;
      const bool kok = kq < 15;
      av[kk] = (kok && i < 15) ? U[i * 15 + kq] : 0.0;
      bv[kk] = !kok ? 0.0 : (bc < 30 ? raw[kq * 30 + bc] : (bc == 30 ? raw[450 + kq] : 0.0));
    }
#pragma unroll
    for (int kk = 0; kk < 4; kk++) dmma(c0, c1, av[kk], bv[kk]);
    if (i < 15) {
      const int j0 = 8 * tj + 2 * q4;
      if (j0 < 30) { fin[i * 30 + j0] = c0; fin[i * 30 + j0 + 1] = c1; }
      else if (j0 == 30) fin[450 + i] = c0;
    }
  }
  __syncwarp();
  auto gcol = [&](int a) -> int {  // local 0..29 -> reduced column
    const int b = a < 6 ? 0 : (a < 15 ? 1 : (a < 21 ? 2 : 3));
    const int o = a < 6 ? a : (a < 15 ? a - 6 : (a < 21 ? a - 15 : a - 21));
    return cols[b] < 0 ? -1 : cols[b] + o;
  };
  // [J r]^T [J r]: 4 x 4 output tiles (rows a < 30; column 30 is the gradient), lower triangle kept
  for (int job = 0; job < 16; job++) {
    const int ta = job >> 2, tb = job & 3;
    const int ar = 8 * ta + g4, bc = 8 * tb + g4;
    double c0 = 0.0, c1 = 0.0, av[4], bv[4];
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      const int kq = 4 * kk + q4;
      const bool kok = kq < 15;
      av[kk] = (kok && ar < 30) ? fin[kq * 30 + ar] : 0.0;
      bv[kk] = !kok ? 0.0 : (bc < 30 ? fin[kq * 30 + bc] : (bc == 30 ? fin[450 + kq] : 0.0));
    }
#pragma unroll
    for (int kk = 0; kk < 4; kk++) dmma(c0, c1, av[kk], bv[kk]);
    if (ar < 30) {
      const int ga = gcol(ar);
      if (ga >= 0) {
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int bo = 8 * tb + 2 * q4 + u;
          const double v = u == 0 ? c0 : c1;
          if (bo < 30) { const int gb = gcol(bo); if (gb >= 0 && gb <= ga && v != 0.0) atomicAdd(&H[(size_t)ga * ld + gb], v); }
          else if (bo == 30) atomicAdd(&g[ga], v);
        }
      }
    }
  }
  double s_ = lane < 15 ? fin[450 + lane] * fin[450 + lane] : 0.0;
  s_ = warp_sum(s_);
  if (lane == 0) atomicAdd(&ctl->cand_cost_misc, 0.5 * s_);
}

// ------------------------------------------------------------------------------------------------
// Fused reprojection linearisation.  One warp = one job (a run of 32-observation tiles of one group).
//   per observation : residual, Jacobians, Huber  ->  landmark-side record {h, g, w_td, w_slot[..]}
//   per group       : [J_slots | (J_td) | r]^T [J_slots | (J_td) | r] accumulated with fp64 tensor-core
//                     MMAs (m8n8k4) from a shared-memory staging tile, flushed with atomics.
// NCT = 8-column tiles of the staged matrix (2: two six-dof slots + r, 4: four slots + td + r)
// KR  = staged rows per observation (2, or 4 for the 3-row depth factor)
template <int NCT, int KR>
__global__ void __launch_bounds__(128) k_proj_lin(Dev d, int eval_cur, int job_begin, int job_count) {
  constexpr int NS = (NCT == 2) ? 2 : 4;
  constexpr int NCOL = NCT * 8;
  constexpr int LDJ = kTile * KR + 4;
  constexpr int ROWS = (KR == 2) ? 2 : 3;
  constexpr int TDCOL = (NCT == 2) ? -1 : 24;
  constexpr int RCOL = (NCT == 2) ? 12 : 25;
  constexpr int NPAIR = NCT * (NCT + 1) / 2;
  constexpr int kWarpDoubles = GC_SIZE + NCOL * LDJ;
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ji = blockIdx.x * 4 + warp;
  if (ji >= job_count) return;
  const Job jb = d.job[job_begin + ji];
  const WinDesc &w = d.win[jb.win];
  Ctl *ctl = d.ctl + jb.win;
  if (ctl->done || (!eval_cur && !ctl->step_valid)) return;
  const int buf = eval_cur ? ctl->cur : 1 - ctl->cur;
  const Group &g = d.grp[jb.grp];
  double *gc = sm + warp * kWarpDoubles;
  double *Js = gc + GC_SIZE;
  const double *x6 = d.x6[buf] + (size_t)w.off6 * 8;
  const double *R6 = d.R6[buf] + (size_t)w.off6 * 12;
  const int type = g.type;
  if (type != PDEPTH) {
    const int bi = g.blk[0], bj = g.blk[1], ba = g.blk[2], bb = g.blk[3];
    build_group_consts(type, bi >= 0 ? R6 + bi * 12 : nullptr, bi >= 0 ? x6 + bi * 8 : nullptr,
                       bj >= 0 ? R6 + bj * 12 : nullptr, bj >= 0 ? x6 + bj * 8 : nullptr, R6 + ba * 12, x6 + ba * 8,
                       bb >= 0 ? R6 + bb * 12 : nullptr, bb >= 0 ? x6 + bb * 8 : nullptr, gc);
  }
  const double td = d.xtd[buf][jb.win];
  const double *xlm = d.xlm[buf] + w.offlm;
  const bool need_ext = g.need_ext, need_td = g.need_td;
  const bool has_cols = (g.slot_src[0] >= 0) || (NS > 2 && g.td_col >= 0);
  double acc[NPAIR][2];
#pragma unroll
  for (int p = 0; p < NPAIR; p++) { acc[p][0] = 0.0; acc[p][1] = 0.0; }
  double cost = 0.0;
  // zero the padding columns of the staging tile once
  for (int c = RCOL + 1; c < NCOL; c++)
    for (int q = 0; q < KR; q++) Js[c * LDJ + lane * KR + q] = 0.0;
  for (int t = 0; t < jb.ntiles; t++) {
    const int tile = jb.tile_begin + t;
    const double *ob = d.obs + (size_t)tile * kObsFields * kTile;
    const int lm = d.obs_lm[(size_t)tile * kTile + lane];
    double f[kObsFields];
#pragma unroll
    for (int k = 0; k < kObsFields; k++) f[k] = ob[k * kTile + lane];
    ProjOut<ROWS> o;
    double lam = lm >= 0 ? xlm[lm] : 1.0;
    if (type == PDEPTH) {
      // OneFrameDepth (depth_factor.h:9-29): r = (lambda - 1/depth) * depth_sqrt_inf, f[20] = 1/depth
#pragma unroll
      for (int q = 0; q < ROWS; q++) { o.r[q] = 0; o.jl[q] = 0; o.jt[q] = 0; }
#pragma unroll
      for (int s = 0; s < 4; s++)
#pragma unroll
        for (int q = 0; q < ROWS; q++)
#pragma unroll
          for (int k = 0; k < 6; k++) o.J[s][q][k] = 0;
      double r0 = (lam - f[20]) * d.prm.depth_sqrt_inf, s2 = r0 * r0, sc = 1.0, hub = d.prm.huber;
      if (hub > 0 && s2 > hub * hub) { double rs = sqrt(s2); o.cost = 0.5 * (2 * hub * rs - hub * hub); sc = sqrt(hub / rs); }
      else o.cost = 0.5 * s2;
      o.r[0] = r0 * sc; o.jl[0] = d.prm.depth_sqrt_inf * sc;
    } else if (need_ext) {
      if (need_td) proj_eval<ROWS, true, true>(type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, d.prm.huber, o);
      else proj_eval<ROWS, true, false>(type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, d.prm.huber, o);
    } else {
      if (need_td) proj_eval<ROWS, false, true>(type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, d.prm.huber, o);
      else proj_eval<ROWS, false, false>(type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, d.prm.huber, o);
    }
    const bool valid = lm >= 0;
    // ---- landmark-side record
    double hl = 0, gl = 0, wtd = 0;
#pragma unroll
    for (int q = 0; q < ROWS; q++) { hl += o.jl[q] * o.jl[q]; gl += o.jl[q] * o.r[q]; if (NS > 2 && need_td) wtd += o.jt[q] * o.jl[q]; }
    // records are stored landmark-major (obs_slot: tile slot -> position in the landmark's run), so the per-landmark
    // reduction streams them; padding lanes (slot -1) never write
    const int rslot = d.obs_slot[(size_t)tile * kTile + lane];
    double *rec = d.rec[buf] + (size_t)w.off_rec + (size_t)(rslot < 0 ? 0 : rslot) * w.rec_stride;
    if (valid) {
      cost += o.cost;
      reinterpret_cast<double2 *>(rec)[0] = make_double2(hl, gl);
      // rec[3] (and rec[28..29] of wide records) carry the reduced-system columns of the slots, so the
      // per-landmark gather needs no group lookup
      reinterpret_cast<double2 *>(rec)[1] = make_double2(wtd, __hiloint2double(g.slot_col[0], g.slot_col[1]));
      if (NS > 2) reinterpret_cast<double2 *>(rec)[14] = make_double2(__hiloint2double(g.slot_col[2], g.slot_col[3]), __hiloint2double(g.td_col, -1));
      else if (w.rec_stride == 32) reinterpret_cast<double2 *>(rec)[14] = make_double2(__hiloint2double(-1, -1), __hiloint2double(-1, -1));
    }
    // ---- slots -> staging tile + coupling vector
#pragma unroll
    for (int s = 0; s < NS; s++) {
      const int src = g.slot_src[s];
      double wv[6];
#pragma unroll
      for (int k = 0; k < 6; k++) {
        double jq[ROWS];
#pragma unroll
        for (int q = 0; q < ROWS; q++) {
          double v = 0.0;
          if (src == 0) v = o.J[0][q][k];
          else if (src == 1) v = o.J[1][q][k];
          else if (src == 2) v = o.J[2][q][k];
          else if (src == 3) v = o.J[3][q][k];
          jq[q] = valid ? v : 0.0;
        }
        double ws = 0;
#pragma unroll
        for (int q = 0; q < ROWS; q++) ws += jq[q] * o.jl[q];
        wv[k] = ws;
        double *dst = Js + (s * 6 + k) * LDJ + lane * KR;
        if (KR == 2) *reinterpret_cast<double2 *>(dst) = make_double2(jq[0], jq[1]);
        else { reinterpret_cast<double2 *>(dst)[0] = make_double2(jq[0], jq[1]); reinterpret_cast<double2 *>(dst)[1] = make_double2(jq[ROWS - 1], 0.0); }
      }
      if (valid && src >= 0) {
        double2 *r2 = reinterpret_cast<double2 *>(rec + 4 + s * 6);
        r2[0] = make_double2(wv[0], wv[1]); r2[1] = make_double2(wv[2], wv[3]); r2[2] = make_double2(wv[4], wv[5]);
      }
    }
    if (NS > 2) {
      double *dst = Js + TDCOL * LDJ + lane * KR;
      double t0 = (valid && need_td) ? o.jt[0] : 0.0, t1 = (valid && need_td) ? o.jt[1] : 0.0;
      if (KR == 2) *reinterpret_cast<double2 *>(dst) = make_double2(t0, t1);
      else { reinterpret_cast<double2 *>(dst)[0] = make_double2(t0, t1); reinterpret_cast<double2 *>(dst)[1] = make_double2((valid && need_td) ? o.jt[ROWS - 1] : 0.0, 0.0); }
    }
    {
      double *dst = Js + RCOL * LDJ + lane * KR;
      double r0 = valid ? o.r[0] : 0.0, r1 = valid ? o.r[1] : 0.0;
      if (KR == 2) *reinterpret_cast<double2 *>(dst) = make_double2(r0, r1);
      else { reinterpret_cast<double2 *>(dst)[0] = make_double2(r0, r1); reinterpret_cast<double2 *>(dst)[1] = make_double2(valid ? o.r[ROWS - 1] : 0.0, 0.0); }
    }
    __syncwarp();
    if (has_cols) {
      // ---- tensor-core accumulation: K = 32*KR staged rows, 4 per MMA
      const int kq = lane & 3, cr = lane >> 2;
#pragma unroll 4
      for (int st = 0; st < kTile * KR / 4; st++) {
        double v[NCT];
#pragma unroll
        for (int c = 0; c < NCT; c++) v[c] = Js[(c * 8 + cr) * LDJ + st * 4 + kq];
        int p = 0;
#pragma unroll
        for (int cm = 0; cm < NCT; cm++)
#pragma unroll
          for (int cn = cm; cn < NCT; cn++) { dmma(acc[p][0], acc[p][1], v[cm], v[cn]); p++; }
      }
    }
    __syncwarp();
  }
  // ---- flush
  cost = warp_sum(cost);
  if (lane == 0) atomicAdd(&ctl->cand_cost_proj, cost);
  if (!has_cols) return;
  double *H = d.Hcc[buf] + w.offH;
  double *gv = d.gc[buf] + w.offc;
  const int ld = w.ldh;
  auto l2g = [&](int m) -> int {
    if (m < NS * 6) { int sc = g.slot_col[m / 6]; return sc < 0 ? -1 : sc + m % 6; }
    if (m == TDCOL) return g.td_col;
    return -1;
  };
  const int row = lane >> 2, c0 = (lane & 3) * 2;
  int p = 0;
#pragma unroll
  for (int cm = 0; cm < NCT; cm++)
#pragma unroll
    for (int cn = cm; cn < NCT; cn++) {
      const int m = cm * 8 + row, gm = l2g(m);
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int n = cn * 8 + c0 + e;
        const double v = acc[p][e];
        if (gm >= 0) {
          if (n == RCOL) atomicAdd(&gv[gm], v);
          else {
            const int gn = l2g(n);
            // Hcc is stored lower-triangular: an off-diagonal tile pair lands once at (max, min); a diagonal tile holds
            // both triangles of its symmetric block, of which the lower one is kept
            if (gn >= 0) {
              if (cm != cn) atomicAdd(&H[(size_t)max(gm, gn) * ld + min(gm, gn)], v);
              else if (gn <= gm) atomicAdd(&H[(size_t)gm * ld + gn], v);
            }
          }
        }
      }
      p++;
    }
}

// explicit instantiations used by the host launcher
template __global__ void k_proj_lin<2, 2>(Dev, int, int, int);
template __global__ void k_proj_lin<4, 2>(Dev, int, int, int);
template __global__ void k_proj_lin<2, 4>(Dev, int, int, int);
template __global__ void k_proj_lin<4, 4>(Dev, int, int, int);

// ------------------------------------------------------------------------------------------------
// Fast path of the fused reprojection linearisation for the dominant case: a two-frame factor (2F1C / 2F2C)
// whose two poses are free and whose extrinsics / td are constant (NCT = 2, KR = 2, slots = {pose_i, pose_j}).
// Same arithmetic as proj_eval<2,false,false>, but the Jacobian rows are emitted straight into the staging tile
// and the landmark record, which keeps the live state small enough for 3 CTAs / SM.
#ifndef D2BA_PP_BLOCKS
#define D2BA_PP_BLOCKS 4
#endif
// The 128-byte landmark records of a tile are staged in shared memory (16-byte units, XOR-swizzled) and written out four
// whole records per store instruction: a lane storing its own record touched 32 different lines per instruction, eight
// times per tile -- that, not DRAM, kept L1/TEX at 70 %.  The landmark index / inverse depth of the next tile are
// fetched during the arithmetic and the DMMA pass of the current one.
constexpr int kPpRows = 13;                          // staged Jacobian rows: 12 + residual (rows 13..15 of the MMA tile read as zero)
constexpr int kPpWarpDoubles = GC_SIZE + kPpRows * (kTile * 2 + 4) + kTile * 16;
static size_t proj_pp_smem() { return (size_t)4 * kPpWarpDoubles * 8; }
template <bool SHIFT0>
__global__ void __launch_bounds__(128, D2BA_PP_BLOCKS) k_proj_lin_pp(Dev d, int eval_cur, int job_begin, int job_count) {
  constexpr int LDJ = kTile * 2 + 4, RCOL = 12;
  extern __shared__ __align__(16) double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ji = blockIdx.x * 4 + warp;
  if (ji >= job_count) return;
  const Job jb = d.job[job_begin + ji];
  const WinDesc &w = d.win[jb.win];
  Ctl *ctl = d.ctl + jb.win;
  if (ctl->done || (!eval_cur && !ctl->step_valid)) return;
  const int buf = eval_cur ? ctl->cur : 1 - ctl->cur;
  const Group &g = d.grp[jb.grp];
  double *gc = sm + warp * kPpWarpDoubles;
  double *Js = gc + GC_SIZE;
  double2 *stg = reinterpret_cast<double2 *>(Js + kPpRows * LDJ);   // [32 records][8 x 16 B], unit (r, c) at r * 8 + (c ^ (r & 7))
  const double *xlm = d.xlm[buf] + w.offlm;
  int lm = d.obs_lm[(size_t)jb.tile_begin * kTile + lane];
  int rslot = d.obs_slot[(size_t)jb.tile_begin * kTile + lane];   // needed only for the record store
  double lam = lm >= 0 ? xlm[lm] : 1.0;
  {
    const double *x6 = d.x6[buf] + (size_t)w.off6 * 8;
    const double *R6 = d.R6[buf] + (size_t)w.off6 * 12;
    const int bi = g.blk[0], bj = g.blk[1], ba = g.blk[2], bb = g.blk[3];
    build_group_consts(g.type, R6 + bi * 12, x6 + bi * 8, R6 + bj * 12, x6 + bj * 8, R6 + ba * 12, x6 + ba * 8,
                       bb >= 0 ? R6 + bb * 12 : nullptr, bb >= 0 ? x6 + bb * 8 : nullptr, gc);
  }
  const double td = d.xtd[buf][jb.win];
  const double s_px = d.prm.sqrt_info_px, huber = d.prm.huber;
  double acc[3][2] = {{0, 0}, {0, 0}, {0, 0}};
  double cost = 0.0;
  const int kq = lane & 3, cr = lane >> 2;
  __syncwarp();
  for (int t = 0; t < jb.ntiles; t++) {
    const int tile = jb.tile_begin + t;
    const bool valid = lm >= 0;
    const double *ob = d.obs + (size_t)tile * kObsFields * kTile + lane;
    double pi[3] = {ob[0 * kTile], ob[1 * kTile], ob[2 * kTile]};
    double pj[3] = {ob[3 * kTile], ob[4 * kTile], ob[5 * kTile]};
    if (!SHIFT0) {
      const double dti = td - ob[12 * kTile], dtj = td - ob[13 * kTile];
#pragma unroll
      for (int k = 0; k < 3; k++) { pi[k] -= dti * ob[(6 + k) * kTile]; pj[k] -= dtj * ob[(9 + k) * kTile]; }
    }
    double B[6];
#pragma unroll
    for (int k = 0; k < 6; k++) B[k] = ob[(14 + k) * kTile];
    int lm_n = -1, rslot_n = -1;
    if (t + 1 < jb.ntiles) {
      lm_n = d.obs_lm[(size_t)(tile + 1) * kTile + lane];
      rslot_n = d.obs_slot[(size_t)(tile + 1) * kTile + lane];
    }
    const double il = 1.0 / lam;
    const double Pci[3] = {pi[0] * il, pi[1] * il, pi[2] * il};
    double Pmi[3], Pmj[3], Pcj[3], tt[3];
    mv3(gc + GC_RA, Pci, Pmi);
    Pmi[0] += gc[GC_TA]; Pmi[1] += gc[GC_TA + 1]; Pmi[2] += gc[GC_TA + 2];
    mv3(gc + GC_RJI, Pmi, Pmj);
    Pmj[0] += gc[GC_TJI]; Pmj[1] += gc[GC_TJI + 1]; Pmj[2] += gc[GC_TJI + 2];
    tt[0] = Pmj[0] - gc[GC_TB]; tt[1] = Pmj[1] - gc[GC_TB + 1]; tt[2] = Pmj[2] - gc[GC_TB + 2];
    mtv3(gc + GC_RB, tt, Pcj);
    const double in = rsqrt(dot3(Pcj, Pcj)), inj = rsqrt(dot3(pj, pj));
    const double ph[3] = {Pcj[0] * in, Pcj[1] * in, Pcj[2] * in};
    const double e[3] = {ph[0] - pj[0] * inj, ph[1] - pj[1] * inj, ph[2] - pj[2] * inj};
    double r0 = s_px * dot3(B, e), r1 = s_px * dot3(B + 3, e);
    const double ss = r0 * r0 + r1 * r1;
    double sc = 1.0, oc = 0.5 * ss;
    if (huber > 0 && ss > huber * huber) { const double rs = sqrt(ss); oc = 0.5 * (2.0 * huber * rs - huber * huber); sc = sqrt(huber / rs); }
    r0 *= sc; r1 *= sc;
    double red[2][3];
    {
      const double b0 = dot3(B, ph), b1 = dot3(B + 3, ph), sn = sc * s_px * in;
#pragma unroll
      for (int k = 0; k < 3; k++) { red[0][k] = sn * (B[k] - b0 * ph[k]); red[1][k] = sn * (B[3 + k] - b1 * ph[k]); }
    }
    // Jacobian rows go straight into the staging tile (K index = q * 32 + lane: conflict-free scalar stores, and the J^T J
    // sums do not care about the order of the K rows) and into the coupling vector; pose_j's position block is minus
    // pose_i's, so only nine of the twelve coupling entries are accumulated.  Keeps the live state small.
    double jl[2];
#pragma unroll
    for (int q = 0; q < 2; q++) { double Dc[3]; rm3(red[q], gc + GC_JC, Dc); jl[q] = -il * dot3(Dc, Pci); }
    if (!valid) { r0 = 0; r1 = 0; jl[0] = 0; jl[1] = 0; red[0][0] = red[0][1] = red[0][2] = red[1][0] = red[1][1] = red[1][2] = 0.0; } else cost += oc;
    double wi[6] = {0, 0, 0, 0, 0, 0}, wjr[3] = {0, 0, 0};
#pragma unroll
    for (int q = 0; q < 2; q++) {
      double A[3], Bm[3], Cr[3], c1[3], c2[3];
      rm3(red[q], gc + GC_JW, A);
      rm3(red[q], gc + GC_JM, Bm);
      Cr[0] = red[q][0] * gc[GC_RB + 0] + red[q][1] * gc[GC_RB + 1] + red[q][2] * gc[GC_RB + 2];
      Cr[1] = red[q][0] * gc[GC_RB + 3] + red[q][1] * gc[GC_RB + 4] + red[q][2] * gc[GC_RB + 5];
      Cr[2] = red[q][0] * gc[GC_RB + 6] + red[q][1] * gc[GC_RB + 7] + red[q][2] * gc[GC_RB + 8];
      cross3(Bm, Pmi, c1);
      cross3(Cr, Pmj, c2);
      double *jq = Js + q * kTile + lane;
#pragma unroll
      for (int k = 0; k < 3; k++) {
        jq[k * LDJ] = A[k]; jq[(3 + k) * LDJ] = -c1[k]; jq[(6 + k) * LDJ] = -A[k]; jq[(9 + k) * LDJ] = c2[k];
        wi[k] = fma(A[k], jl[q], wi[k]); wi[3 + k] = fma(-c1[k], jl[q], wi[3 + k]); wjr[k] = fma(c2[k], jl[q], wjr[k]);
      }
    }
    Js[RCOL * LDJ + lane] = r0; Js[RCOL * LDJ + kTile + lane] = r1;
    // records are stored landmark-major (obs_slot: tile slot -> position in the landmark's run), so the per-landmark
    // reduction streams them; padding lanes (slot -1) never write
    {
      double2 *sr = stg + lane * 8;
      const int sw = lane & 7;
      sr[0 ^ sw] = make_double2(jl[0] * jl[0] + jl[1] * jl[1], jl[0] * r0 + jl[1] * r1);
      sr[1 ^ sw] = make_double2(0.0, __hiloint2double(g.slot_col[0], g.slot_col[1]));
      sr[2 ^ sw] = make_double2(wi[0], wi[1]); sr[3 ^ sw] = make_double2(wi[2], wi[3]); sr[4 ^ sw] = make_double2(wi[4], wi[5]);
      sr[5 ^ sw] = make_double2(-wi[0], -wi[1]); sr[6 ^ sw] = make_double2(-wi[2], wjr[0]); sr[7 ^ sw] = make_double2(wjr[1], wjr[2]);
    }
    const int my_slot = valid ? rslot : -1;
    lm = lm_n; rslot = rslot_n;
    lam = lm >= 0 ? xlm[lm] : 1.0;                    // next tile's inverse depth: in flight during the MMA pass
    __syncwarp();
    {
      // four whole records per store instruction: lanes 8k .. 8k+7 write the 128 contiguous bytes of record 4 j + k
      double *recs = d.rec[buf] + (size_t)w.off_rec;
      const int c = lane & 7, stride = w.rec_stride;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int r = 4 * j + (lane >> 3);
        const int slot = __shfl_sync(0xffffffffu, my_slot, r);
        if (slot >= 0) {
          double2 *dst = reinterpret_cast<double2 *>(recs + (size_t)slot * stride);
          dst[c] = stg[r * 8 + (c ^ (r & 7))];
          if (stride == 32 && c == 0) dst[14] = make_double2(__hiloint2double(-1, -1), __hiloint2double(-1, -1));
        }
      }
    }
#pragma unroll 4
    for (int st = 0; st < kTile * 2 / 4; st++) {
      const double v0 = Js[cr * LDJ + st * 4 + kq], v1 = cr < kPpRows - 8 ? Js[(8 + cr) * LDJ + st * 4 + kq] : 0.0;
      dmma(acc[0][0], acc[0][1], v0, v0);
      dmma(acc[1][0], acc[1][1], v0, v1);
      dmma(acc[2][0], acc[2][1], v1, v1);
    }
    __syncwarp();
  }
  cost = warp_sum(cost);
  if (lane == 0) atomicAdd(&ctl->cand_cost_proj, cost);
  double *H = d.Hcc[buf] + w.offH;
  double *gv = d.gc[buf] + w.offc;
  const int ld = w.ldh, ci = g.slot_col[0], cj = g.slot_col[1];
  auto l2g = [&](int m) -> int { return m < 6 ? ci + m : (m < 12 ? cj + m - 6 : -1); };
  const int row = lane >> 2, c0 = (lane & 3) * 2;
#pragma unroll
  for (int p = 0; p < 3; p++) {
    const int cm = p == 2 ? 1 : 0, cn = p == 0 ? 0 : 1;
    const int m = cm * 8 + row, gm = l2g(m);
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int n = cn * 8 + c0 + e;
      const double v = acc[p][e];
      if (gm >= 0) {
        if (n == RCOL) atomicAdd(&gv[gm], v);
        else {
          const int gn = l2g(n);
          if (gn >= 0) {   // lower-triangular storage (see k_proj_lin)
            if (cm != cn) atomicAdd(&H[(size_t)max(gm, gn) * ld + min(gm, gn)], v);
            else if (gn <= gm) atomicAdd(&H[(size_t)gm * ld + gn], v);
          }
        }
      }
    }
  }
}
template __global__ void k_proj_lin_pp<true>(Dev, int, int, int);
template __global__ void k_proj_lin_pp<false>(Dev, int, int, int);

// debug: raw (un-robustified) residual + full 3x26 Jacobian per observation tile slot
__global__ void k_proj_debug(Dev d, double *out /*[tiles*32][81]*/, int n_tiles_total, const int *tile_win) {
  const int tile = blockIdx.x;
  if (tile >= n_tiles_total) return;
  const int lane = threadIdx.x & 31;
  __shared__ double gc[GC_SIZE];
  const int wi = tile_win[tile];
  const WinDesc &w = d.win[wi];
  const int buf = d.ctl[wi].cur;
  const Group &g = d.grp[d.tile_grp[tile]];
  const double *x6 = d.x6[buf] + (size_t)w.off6 * 8;
  const double *R6 = d.R6[buf] + (size_t)w.off6 * 12;
  const double *ob = d.obs + (size_t)tile * kObsFields * kTile;
  const int lm = d.obs_lm[(size_t)tile * kTile + lane];
  double f[kObsFields];
  for (int k = 0; k < kObsFields; k++) f[k] = ob[k * kTile + lane];
  double *rec = out + ((size_t)tile * kTile + lane) * 81;
  for (int k = 0; k < 81; k++) rec[k] = 0.0;
  double lam = lm >= 0 ? d.xlm[buf][w.offlm + lm] : 1.0;
  if (g.type == PDEPTH) {
    if (lm >= 0) { rec[0] = (lam - f[20]) * d.prm.depth_sqrt_inf; rec[3 + 24] = d.prm.depth_sqrt_inf; }
    return;
  }
  const int bi = g.blk[0], bj = g.blk[1], ba = g.blk[2], bb = g.blk[3];
  build_group_consts(g.type, bi >= 0 ? R6 + bi * 12 : nullptr, bi >= 0 ? x6 + bi * 8 : nullptr, bj >= 0 ? R6 + bj * 12 : nullptr,
                     bj >= 0 ? x6 + bj * 8 : nullptr, R6 + ba * 12, x6 + ba * 8, bb >= 0 ? R6 + bb * 12 : nullptr,
                     bb >= 0 ? x6 + bb * 8 : nullptr, gc);
  if (lm < 0) return;
  ProjOut<3> o;
  o.r[2] = 0; o.jl[2] = 0; o.jt[2] = 0;
  const double td = d.xtd[buf][wi];
  if (g.type == P2F1CD) proj_eval<3, true, true>(g.type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, -1.0, o);
  else {
    ProjOut<2> o2;
    proj_eval<2, true, true>(g.type, gc, f, lam, td, d.prm.sqrt_info_px, d.prm.depth_sqrt_inf, -1.0, o2);
    for (int q = 0; q < 2; q++) { o.r[q] = o2.r[q]; o.jl[q] = o2.jl[q]; o.jt[q] = o2.jt[q]; for (int s = 0; s < 4; s++) for (int k = 0; k < 6; k++) o.J[s][q][k] = o2.J[s][q][k]; }
    for (int s = 0; s < 4; s++) for (int k = 0; k < 6; k++) o.J[s][2][k] = 0;
  }
  const int rows = g.type == P2F1CD ? 3 : 2;
  for (int q = 0; q < rows; q++) {
    rec[q] = o.r[q];
    double *Jr = rec + 3 + q * 26;
    for (int s = 0; s < 4; s++) {
      bool present = (s < 2) ? (g.type != P1F2C) : (s == 2 ? true : (g.type == P2F2C || g.type == P1F2C));
      for (int k = 0; k < 6; k++) Jr[s * 6 + k] = present ? o.J[s][q][k] : 0.0;
    }
    Jr[24] = o.jl[q]; Jr[25] = o.jt[q];
  }
}

// debug: whitened residual + Jacobian of every IMU factor (one thread per factor), same imu_raw as k_misc_lin
__global__ void k_imu_debug(Dev d, double *out /*[n_imu_total][465]*/, const int *imu_win, int n_imu_total) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_imu_total) return;
  const int wi = imu_win[f];
  const WinDesc &w = d.win[wi];
  const int buf = d.ctl[wi].cur;
  const double *x6 = d.x6[buf] + (size_t)w.off6 * 8, *xsb = d.xsb[buf] + (size_t)w.offsb * 9;
  const ImuDesc &im = d.imu[f];
  double raw[465];
  for (int i = 0; i < 465; i++) raw[i] = 0.0;
  imu_raw(d.imu_c + (size_t)f * kImuStride, x6 + im.pi * 8, xsb + im.si * 9, x6 + im.pj * 8, xsb + im.sj * 9, d.prm.gravity, raw + 450, raw);
  const double *U = d.imu_U + (size_t)f * 225;
  double *o = out + (size_t)f * 465;
  for (int i = 0; i < 15; i++) {
    double s = 0; for (int k = 0; k < 15; k++) s += U[i * 15 + k] * raw[450 + k];
    o[i] = s;
    for (int j = 0; j < 30; j++) { double a = 0; for (int k = 0; k < 15; k++) a += U[i * 15 + k] * raw[k * 30 + j]; o[15 + i * 30 + j] = a; }
  }
}
__global__ void k_cons_debug(Dev d, double *out /*[n6_total][62]*/, const int *blk_win, int n6_total) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n6_total) return;
  double *o = out + (size_t)b * 62;
  for (int i = 0; i < 62; i++) o[i] = 0.0;
  if (d.slot6[b] < 0) return;
  const int wi = blk_win[b];
  const double *x = d.x6[d.ctl[wi].cur] + (size_t)b * 8, *z = d.z6 + (size_t)b * 8, *tl = d.tilde6 + (size_t)b * 6;
  double r[6], Rz[9], L3[9];
  const double wq = d.prm.rho_T, wT = d.prm.rho_theta;
  cons_eval(x, z, tl, wq, wT, r, Rz, L3);
  for (int i = 0; i < 7; i++) { o[i] = x[i]; o[7 + i] = z[i]; }
  for (int i = 0; i < 6; i++) { o[14 + i] = tl[i]; o[20 + i] = r[i]; }
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { o[26 + i * 6 + j] = wT * Rz[j * 3 + i]; o[26 + (3 + i) * 6 + 3 + j] = wq * L3[i * 3 + j]; }
}
void launch_imu_debug(const Dev &d, double *out, const int *imu_win, int n, cudaStream_t s) { if (n > 0) k_imu_debug<<<(n + 31) / 32, 32, 0, s>>>(d, out, imu_win, n); }
void launch_cons_debug(const Dev &d, double *out, const int *blk_win, int n, cudaStream_t s) { if (n > 0) k_cons_debug<<<(n + 63) / 64, 64, 0, s>>>(d, out, blk_win, n); }

// ------------------------------------------------------------------------------------------------
// Per-landmark reduction, wide records (warp per landmark; compact records: k_lm_gather16 below).  The landmark's
// records are visited serially, the 32 record entries in parallel across lanes, so there are no write conflicts and
// the result is deterministic.  Output: Wt[l][0..n_lc) = w_l / sqrt(h'), Wt[l][n_lc] = g_l / sqrt(h'),
// h' = h_l + mu D_l^2.
// position of W-space column `col` in a row buffer that holds only the 32-column tiles named by `mask` (ascending)
D2BA_DEV int row_slot(unsigned long long mask, int col) { return __popcll(mask & ((1ull << (col >> 5)) - 1ull)) * 32 + (col & 31); }
constexpr int kGatherWarps = 8;
__global__ void __launch_bounds__(kGatherWarps * 32) k_lm_gather(Dev d, const int *lm_win, int n_lm_total, int max_ldw) {
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gl_idx = blockIdx.x * kGatherWarps + warp;
  if (gl_idx >= n_lm_total) return;
  const int wi = lm_win[gl_idx];
  const WinDesc &w = d.win[wi];
  if (w.rec_stride == 16) return;   // compact windows: k_lm_gather16
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse) return;
  const int buf = ctl->cur;
  const int l = gl_idx - w.offlm;
  double *row = sm + warp * max_ldw;
  const int nlc = w.n_lc;
  // column tiles (32 wide) this landmark's coupling row touches; windows without leaves (single drone) treat the row as dense
  const unsigned long long mask = w.n_leaf ? d.lm_mask[gl_idx] : ((2ull << (w.n_lc / 32)) - 1ull);
  const int nrt = __popcll(mask);   // the row buffer holds just these tiles, packed
  for (int k = 0; k < nrt; k++) row[k * 32 + lane] = 0.0;
  __syncwarp();
  const int *ptr = d.lm_ptr + w.off_lmptr;
  const double *recs = d.rec[buf] + (size_t)w.off_rec;
  double h = 0, g = 0;
  const int kb = ptr[l], ke = ptr[l + 1];
  // wide records (256 B: extrinsics / td free): one warp load per record, two records in flight
  for (int k0 = kb; k0 < ke; k0 += 32) {
    const int cnt = min(32, ke - k0);
    for (int q = 0; q < cnt; q += 2) {
      const int p0 = k0 + q, p1 = k0 + min(q + 1, cnt - 1);
      const bool two = q + 1 < cnt;
      double v0 = recs[(size_t)p0 * 32 + lane];
      double v1 = two ? recs[(size_t)p1 * 32 + lane] : 0.0;
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const double v = u == 0 ? v0 : v1;
        if (u == 1 && !two) break;
        if (lane == 0) h += v;
        if (lane == 1) g += v;
        const double c01 = __shfl_sync(0xffffffffu, v, 3), c23 = __shfl_sync(0xffffffffu, v, 28), ctd = __shfl_sync(0xffffffffu, v, 29);
        int col = -1;
        if (lane >= 4 && lane < 16) { int sc = lane < 10 ? __double2hiint(c01) : __double2loint(c01); if (sc >= 0) col = sc + (lane - 4) % 6; }
        if (lane >= 16 && lane < 28) { int sc = lane < 22 ? __double2hiint(c23) : __double2loint(c23); if (sc >= 0) col = sc + (lane - 4) % 6; }
        if (lane == 2) col = __double2hiint(ctd);
        if (col >= 0) row[row_slot(mask, col)] += v;
        __syncwarp();
      }
    }
  }
  h = __shfl_sync(0xffffffffu, h, 0);
  g = __shfl_sync(0xffffffffu, g, 1);
  if (w.admm_on) {
    double rl = d.prm.rho_landmark;
    h += rl * rl;
    g += rl * rl * (d.xlm[buf][w.offlm + l] - d.lm_ref[w.offlm + l]);
  }
  const double dl2 = d2_of(h);
  const double hp = h + ctl->mu * dl2;
  const double di = 1.0 / sqrt(hp);
  double *Wt = d.Wt + w.offW + (size_t)l * w.ldw;
  const double *uc = d.uc + w.offc;
  double wu = 0;
  int kk = 0;
  for (unsigned long long m = mask; m; m &= m - 1, kk++) {   // the other tiles of the row stay zero (finalize-time memset)
    const int c = (__ffsll((long long)m) - 1) * 32 + lane;
    if (c >= w.ldw) continue;
    double rv = (c < nlc) ? row[kk * 32 + lane] : 0.0;
    Wt[c] = (c < nlc) ? rv * di : (c == nlc ? g * di : 0.0);
    if (c < nlc) wu += rv * uc[c];
  }
  wu = warp_sum(wu);
  if (lane == 0) {
    d.hl[w.offlm + l] = h; d.gl[w.offlm + l] = g; d.dinv[w.offlm + l] = di; d.wu[w.offlm + l] = wu; d.D2l[w.offlm + l] = dl2;
    if (!(hp > 0.0)) ctl->chol_fail = 1;
    atomicMax(&ctl->gmax_l_bits, (unsigned long long)__double_as_longlong(fabs(g)));
  }
}

// Compact-record windows (rec_stride == 16): one HALF-warp per landmark -- a 128-byte record is exactly one 16-lane
// load, so the two halves of a warp work on two landmarks independently (no cross-half ordering, half-warp masks).
constexpr int kG16Lm = 16;   // landmarks per 256-thread CTA
__global__ void __launch_bounds__(kG16Lm * 16) k_lm_gather16(Dev d, const int *lm_win, int n_lm_total, int max_ldw) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, hw = threadIdx.x >> 4, sub = lane & 15, hbase = lane & 16;
  const unsigned hmask = 0xffffu << hbase;
  const int gl_idx = blockIdx.x * kG16Lm + hw;
  if (gl_idx >= n_lm_total) return;
  const int wi = lm_win[gl_idx];
  const WinDesc &w = d.win[wi];
  if (w.rec_stride != 16) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse) return;
  const int buf = ctl->cur;
  const int l = gl_idx - w.offlm;
  double *row = sm + hw * max_ldw;
  const int nlc = w.n_lc;
  // column tiles (32 wide) this landmark's coupling row touches; windows without leaves (single drone) treat the row as dense
  const unsigned long long mask = w.n_leaf ? d.lm_mask[gl_idx] : ((2ull << (w.n_lc / 32)) - 1ull);
  const int nrt = __popcll(mask);   // the row buffer holds just these tiles, packed
  for (int k = sub; k < nrt * 32; k += 16) row[k] = 0.0;
  __syncwarp(hmask);
  const int *ptr = d.lm_ptr + w.off_lmptr;
  const double *recs = d.rec[buf] + (size_t)w.off_rec;
  double h = 0, g = 0;
  const int kb = ptr[l], ke = ptr[l + 1];
  for (int k0 = kb; k0 < ke; k0 += 8) {   // the landmark's records are contiguous (landmark-major store of k_proj_lin)
    const int cnt = min(8, ke - k0);
    double v[8];
#pragma unroll
    for (int q = 0; q < 8; q++) v[q] = (q < cnt) ? recs[(size_t)(k0 + q) * 16 + sub] : 0.0;
    if (w.gather_nosync) {
      // a column block is only ever named by ONE slot position within this landmark's records (host-checked): a row entry
      // is always updated by the same lane, in program order -- no barrier between records, the updates pipeline
#pragma unroll
      for (int q = 0; q < 8; q++) {
        if (q >= cnt) break;
        const double c01 = __shfl_sync(hmask, v[q], hbase | 3);   // packed column word of the record
        int col = -1;
        if (sub >= 4) { const int sc = sub < 10 ? __double2hiint(c01) : __double2loint(c01); if (sc >= 0) col = sc + (sub - 4) % 6; }
        if (sub == 0) h += v[q];
        if (sub == 1) g += v[q];
        if (col >= 0) row[w.n_leaf ? row_slot(mask, col) : col] += v[q];
      }
    } else {
#pragma unroll
      for (int q = 0; q < 8; q++) {
        if (q >= cnt) break;
        const double c01 = __shfl_sync(hmask, v[q], hbase | 3);   // packed column word of the record
        int col = -1;
        if (sub >= 4) { const int sc = sub < 10 ? __double2hiint(c01) : __double2loint(c01); if (sc >= 0) col = sc + (sub - 4) % 6; }
        if (sub == 0) h += v[q];
        if (sub == 1) g += v[q];
        if (col >= 0) row[row_slot(mask, col)] += v[q];
        __syncwarp(hmask);   // the two slots of different records may name the same column block
      }
    }
  }
  __syncwarp(hmask);
  h = __shfl_sync(hmask, h, hbase);
  g = __shfl_sync(hmask, g, hbase | 1);
  if (w.admm_on) {
    const double rl = d.prm.rho_landmark;
    h += rl * rl;
    g += rl * rl * (d.xlm[buf][w.offlm + l] - d.lm_ref[w.offlm + l]);
  }
  const double dl2 = d2_of(h);
  const double hp = h + ctl->mu * dl2;
  const double di = 1.0 / sqrt(hp);
  double *Wt = d.Wt + w.offW + (size_t)l * w.ldw;
  const double *uc = d.uc + w.offc;
  double wu = 0;
  int kk = 0;
  for (unsigned long long m = mask; m; m &= m - 1, kk++) {   // the other tiles of the row stay zero (finalize-time memset)
    const int c0 = (__ffsll((long long)m) - 1) * 32 + sub;
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int c = c0 + 16 * u;
      if (c >= w.ldw) continue;
      const double rv = (c < nlc) ? row[kk * 32 + sub + 16 * u] : 0.0;
      Wt[c] = (c < nlc) ? rv * di : (c == nlc ? g * di : 0.0);
      if (c < nlc) wu += rv * uc[c];
    }
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) wu += __shfl_xor_sync(hmask, wu, o);
  if (sub == 0) {
    d.hl[w.offlm + l] = h; d.gl[w.offlm + l] = g; d.dinv[w.offlm + l] = di; d.wu[w.offlm + l] = wu; d.D2l[w.offlm + l] = dl2;
    if (!(hp > 0.0)) ctl->chol_fail = 1;
    atomicMax(&ctl->gmax_l_bits, (unsigned long long)__double_as_longlong(fabs(g)));
  }
}

// ------------------------------------------------------------------------------------------------
// Reduced camera system.  Tile list entries: kind 0 = SYRK tile in W-space (32x32), kind 1 = copy tile
// (rows/cols of the speed-bias part, which have no landmark coupling).
// (SchurTile: d2ba_types.cuh.)  Each tile sums over its own list of 32-row chunks of Wt -- the chunks in which some row has
// entries in both column tiles (block sparsity of the landmark rows in multi-agent windows).  kind 2 tiles run before the
// leaf elimination and store only entries in leaf columns (c < hub0), kind 0 tiles after it and store the hub x hub part.
constexpr int kSyrkK = 32;
constexpr int kSyrkLd = 36;  // == 4 (mod 16): conflict-free fragment loads
__global__ void __launch_bounds__(128) k_schur(Dev d, const SchurTile *tiles) {
  const SchurTile t = tiles[blockIdx.x];
  const WinDesc &w = d.win[t.win];
  Ctl *ctl = d.ctl + t.win;
  if (ctl->done || ctl->reuse) return;
  const int buf = ctl->cur;
  const int n = w.n_c, nlc = w.n_lc, ld = w.ldh;
  const double mu = ctl->mu;
  const double *H = d.Hcc[buf] + w.offH;
  const double *gcv = d.gc[buf] + w.offc;
  double *S = d.S + w.offH;
  const int tid = threadIdx.x;
  const double *ucv = d.uc + w.offc;
  const double *D2v = d.D2c + w.offc;
  __shared__ double As[kSyrkK * kSyrkLd], Bs[kSyrkK * kSyrkLd];
  __shared__ double redq[40];
  double uhu = 0.0;   // this tile's share of u^T Hcc u (lower elements, off-diagonal counted twice)
  if (t.kind == 1) {
    // plain copy region: S[i][j] = H[i][j] + mu D^2 (i == j) for i in [nlc, n), j <= i; rhs row j in [nlc, n)
    if (w.sb_elim) return;   // the speed-bias rows were eliminated by k_sb_elim (which also took their share of u^T H u)
    const int i0 = t.tm * 32, j0 = t.tn * 32;
    for (int e = tid; e < 1024; e += 128) {
      int i = i0 + e / 32, j = j0 + e % 32;
      if (i < n && j <= i && i >= nlc) {
        double v = H[(size_t)i * ld + j];
        uhu += (i == j ? 1.0 : 2.0) * v * ucv[i] * ucv[j];
        if (i == j) v += mu * D2v[i];
        S[(size_t)i * ld + j] = v;
      }
      if (i == n && j < n && j >= nlc) S[(size_t)n * ld + j] = gcv[j];
    }
    uhu = block_sum(uhu, redq);
    if (tid == 0 && uhu != 0.0) atomicAdd(&ctl->uHu_cam, uhu);
    return;
  }
  const int warp = tid >> 5, lane = tid & 31;
  const int m0 = t.tm * 32, n0 = t.tn * 32;   // W-space offsets (0..nlc inclusive is valid)
  const int wm = (warp >> 1) * 16, wn = (warp & 1) * 16;
  double acc[2][2][2] = {};
  const double *Wt = d.Wt + w.offW;
  const int ldw = w.ldw;
  const int kq = lane & 3, cr = lane >> 2;
  const int *chunks = d.schur_chunks + t.cb;
  for (int ci = 0; ci < t.cn; ci++) {   // landmark rows, then (hub tiles) the eliminated speed-bias / leaf rows Y
    const int k0 = chunks[ci] * kSyrkK;
    for (int e = tid; e < kSyrkK * 32; e += 128) {
      int k = e / 32, c = e % 32;
      const double *rowp = Wt + (size_t)(k0 + k) * ldw;
      As[k * kSyrkLd + c] = (m0 + c < ldw) ? rowp[m0 + c] : 0.0;
      Bs[k * kSyrkLd + c] = (n0 + c < ldw) ? rowp[n0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < kSyrkK; ks += 4) {
      double a0 = As[(ks + kq) * kSyrkLd + wm + cr], a1 = As[(ks + kq) * kSyrkLd + wm + 8 + cr];
      double b0 = Bs[(ks + kq) * kSyrkLd + wn + cr], b1 = Bs[(ks + kq) * kSyrkLd + wn + 8 + cr];
      dmma(acc[0][0][0], acc[0][0][1], a0, b0);
      dmma(acc[0][1][0], acc[0][1][1], a0, b1);
      dmma(acc[1][0][0], acc[1][0][1], a1, b0);
      dmma(acc[1][1][0], acc[1][1][1], a1, b1);
    }
    __syncthreads();
  }
  // epilogue: W-space (m, c) -> S-space; index nlc of W-space is the rhs row n of S
  const int hub0 = w.hub0;
  const bool leaf_stage = t.kind == 2;
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 2; b++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        int m = m0 + wm + a * 8 + cr, c = n0 + wn + b * 8 + kq * 2 + e;
        double v = acc[a][b][e];
        if ((c < hub0) != leaf_stage) continue;   // a tile straddling the leaf / hub boundary is visited in both stages
        if (m < nlc && c <= m) {
          double hv = H[(size_t)m * ld + c];
          uhu += (m == c ? 1.0 : 2.0) * hv * ucv[m] * ucv[c];
          if (m == c) hv += mu * D2v[m];
          S[(size_t)m * ld + c] = hv - v;
        } else if (m == nlc && c < nlc) {
          S[(size_t)(w.sb_elim ? nlc : n) * ld + c] = gcv[c] - v;   // rhs row of the system the Cholesky will see
        }
      }
  uhu = block_sum(uhu, redq);
  if (tid == 0 && uhu != 0.0) atomicAdd(&ctl->uHu_cam, uhu);
}

// ------------------------------------------------------------------------------------------------
// One-CTA-per-window Schur complement for small landmark-coupled parts (n_lc + 1 <= 96, e.g. the 11-pose
// single-drone window: 67 columns = 9 blocks of 8 -> 45 lower 8x8 blocks instead of 6 padded 32x32 tiles).
// The Wt chunk is staged once per 32 landmarks and shared by all blocks; each warp owns up to kSsMaxB blocks.
constexpr int kSsThreads = 256;
constexpr int kSsMaxB = 10;   // 12*13/2 = 78 lower blocks over 8 warps
__global__ void __launch_bounds__(kSsThreads, 2) k_schur_small(Dev d) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  if (!w.schur_small && !w.hub_small) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse) return;
  const int buf = ctl->cur;
  // window of W-space columns this kernel forms: everything (single-drone window) or the hub [hub0, n_lc] behind the leaves;
  // below, nlc / ldw / the pointers are all relative to that window
  const int c0 = w.hub_small ? w.hub0 : 0;
  const int n = w.n_c - c0, nlc = w.n_lc - c0, ld = w.ldh, ldw = w.hub_small ? ((nlc + 1 + 7) & ~7) : w.ldw, ldwg = w.ldw;
  const double mu = ctl->mu;
  const double *H = d.Hcc[buf] + w.offH + (size_t)c0 * ld + c0;
  const double *gcv = d.gc[buf] + w.offc + c0;
  const double *ucv = d.uc + w.offc + c0, *D2v = d.D2c + w.offc + c0;
  double *S = d.S + w.offH + (size_t)c0 * ld + c0;
  const double *Wt = d.Wt + w.offW + c0;
  extern __shared__ double sm[];
  const int ldws = ldw + 4;
  double *Ws = sm;                            // 2 buffers x 32 x ldws (TMA bulk staged)
  double *redq = sm + 2 * 32 * ldws;          // 40
  __shared__ unsigned long long bar[2];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, kq = lane & 3, cr = lane >> 2;
  const int nb8 = ldw >> 3, nblk = nb8 * (nb8 + 1) / 2;
  int bi[kSsMaxB], bj[kSsMaxB];
  double acc[kSsMaxB][2];
#pragma unroll
  for (int q = 0; q < kSsMaxB; q++) {
    int t = warp + q * 8;
    int i = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);
    while ((i + 1) * (i + 2) / 2 <= t) i++;
    while (i * (i + 1) / 2 > t) i--;
    bi[q] = i; bj[q] = t - i * (i + 1) / 2;
    acc[q][0] = 0.0; acc[q][1] = 0.0;
  }
  const int nq = warp < nblk ? (nblk - 1 - warp) / 8 + 1 : 0;   // blocks owned by this warp (t = warp, warp + 8, ...)
  double uhu = 0.0;
  if (nlc > 0) {
    const int nchunk = w.wt_rows / 32;   // landmark rows, then the eliminated speed-bias rows Y
    const unsigned row_bytes = (unsigned)ldw * 8u;
    if (tid == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); mbar_fence_init(); }
    __syncthreads();
    // producer: one thread issues 32 row copies per chunk (rows are padded in shared memory for conflict-free fragments)
    auto issue = [&](int c, int b) {
      mbar_expect_tx(&bar[b], 32u * row_bytes);
      const double *src = Wt + (size_t)c * 32 * ldwg;
      double *dst = Ws + b * 32 * ldws;
      for (int k = 0; k < 32; k++) bulk_g2s(dst + k * ldws, src + (size_t)k * ldwg, row_bytes, &bar[b]);
    };
    if (tid == 0) { issue(0, 0); if (nchunk > 1) issue(1, 1); }
    for (int c = 0; c < nchunk; c++) {
      const int b = c & 1;
      mbar_wait(&bar[b], (unsigned)((c >> 1) & 1));
      const double *Wb = Ws + b * 32 * ldws;
      // the number of blocks this warp owns is warp-uniform: dispatch once per chunk to a fully unrolled body whose MMAs
      // are unconditional (a predicated mma.sync costs a WARPSYNC each); operands first, then the MMAs back to back
      auto body = [&](auto NQ) {
        constexpr int nq_c = decltype(NQ)::value;
#pragma unroll 2
        for (int ks = 0; ks < 32; ks += 4) {
          const double *wr = Wb + (ks + kq) * ldws + cr;
          double fa[nq_c > 0 ? nq_c : 1], fb[nq_c > 0 ? nq_c : 1];
#pragma unroll
          for (int q = 0; q < nq_c; q++) { fa[q] = wr[bi[q] * 8]; fb[q] = wr[bj[q] * 8]; }
#pragma unroll
          for (int q = 0; q < nq_c; q++) dmma(acc[q][0], acc[q][1], fa[q], fb[q]);
        }
      };
      switch (nq) {
        case 1: body(std::integral_constant<int, 1>()); break;
        case 2: body(std::integral_constant<int, 2>()); break;
        case 3: body(std::integral_constant<int, 3>()); break;
        case 4: body(std::integral_constant<int, 4>()); break;
        case 5: body(std::integral_constant<int, 5>()); break;
        case 6: body(std::integral_constant<int, 6>()); break;
        case 7: body(std::integral_constant<int, 7>()); break;
        case 8: body(std::integral_constant<int, 8>()); break;
        case 9: body(std::integral_constant<int, 9>()); break;
        case 10: body(std::integral_constant<int, 10>()); break;
        default: break;
      }
      __syncthreads();
      if (tid == 0 && c + 2 < nchunk) { fence_proxy_async(); issue(c + 2, b); }
    }
#pragma unroll
    for (int q = 0; q < kSsMaxB; q++) {
      if (warp + q * 8 >= nblk) continue;
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int m = bi[q] * 8 + cr, c = bj[q] * 8 + kq * 2 + e;
        const double v = acc[q][e];
        if (m < nlc && c <= m) {
          double hv = H[(size_t)m * ld + c];
          uhu += (m == c ? 1.0 : 2.0) * hv * ucv[m] * ucv[c];
          if (m == c) hv += mu * D2v[m];
          S[(size_t)m * ld + c] = hv - v;
        } else if (m == nlc && c < nlc) {
          S[(size_t)(w.sb_elim ? nlc : n) * ld + c] = gcv[c] - v;   // rhs row of the system the Cholesky will see
        }
      }
    }
  }
  // rows of the speed-bias part (no landmark coupling) and the rest of the rhs row; when the shared-memory
  // Cholesky owns this window it reads them straight from Hcc instead (saves the copy through S)
  const int nrow = (w.chol_smem || w.sb_elim) ? 0 : n - nlc;
  for (int e = tid; e < nrow * n; e += kSsThreads) {
    const int i = nlc + e / n, j = e % n;
    if (j > i) continue;
    double v = H[(size_t)i * ld + j];
    uhu += (i == j ? 1.0 : 2.0) * v * ucv[i] * ucv[j];
    if (i == j) v += mu * D2v[i];
    S[(size_t)i * ld + j] = v;
  }
  if (!w.chol_smem && !w.sb_elim) for (int j = nlc + tid; j < n; j += kSsThreads) S[(size_t)n * ld + j] = gcv[j];
  uhu = block_sum(uhu, redq);
  if (tid == 0) atomicAdd(&ctl->uHu_cam, uhu);
}

// ------------------------------------------------------------------------------------------------
// Blocked bordered Cholesky of the reduced system, one CTA per window.
// S is (n+1) x ld row-major, lower part valid; row n carries the right-hand side, so after the
// factorisation it holds y = L^-1 g ("forward substitution for free").  Back substitution then gives
// the Gauss-Newton camera step dc = -L^-T y.
// Per 32-column panel: (a) warp 0 factors the 32x32 diagonal block in shared memory (one row per lane),
// (b) every remaining row is solved against it by its own thread (TRSM, registers), (c) the trailing
// matrix is updated with 4x4 register tiles.  Only two block barriers per panel phase.
constexpr int kCholThreads = 256;
constexpr int kNB = 32;
__global__ void __launch_bounds__(kCholThreads) k_chol(Dev d, int max_rows) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  Ctl *ctl = d.ctl + wi;
  if (w.chol_smem) return;
  if (ctl->done || ctl->reuse) return;
  if (ctl->chol_fail) return;
  extern __shared__ double sm[];
  const int ldp = max_rows + 4;     // panel stored transposed: Pt[c][r]
  double *Pt = sm;                  // kNB * ldp
  double *xs = sm + kNB * ldp;      // solution / scratch (max_rows)
  double *redb = xs + max_rows + 8; // 16 x 32 partial sums
  double *Dg = redb + 16 * 32;      // kNB x (kNB+1) diagonal block (row-major, lower)
  double *invd = Dg + kNB * (kNB + 1);  // reciprocal diagonal of L, all n columns
  __shared__ int fail;
  // speed-bias blocks / leaves eliminated beforehand: the dense part is the hub [hub0, n_lc) with the rhs in row n_lc
  const bool reduced = w.sb_elim || w.n_leaf > 0;
  const int c0 = reduced ? w.hub0 : 0;
  const int n = reduced ? w.n_hub : w.n_c, n1 = n + 1, ld = w.ldh;
  double *S = d.S + w.offH + (size_t)c0 * ld + c0;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) fail = 0;
  __syncthreads();
  for (int k0 = 0; k0 < n; k0 += kNB) {
    const int nb = min(kNB, n - k0), nr = n1 - k0;
    // load panel (rows k0..n, cols k0..k0+nb); diagonal block also into Dg (identity padded)
    for (int e = tid; e < nr * kNB; e += nt) {
      int r = e / kNB, c = e % kNB;
      double v = (c < nb) ? S[(size_t)(k0 + r) * ld + k0 + c] : 0.0;
      Pt[c * ldp + r] = v;
      if (r < kNB) Dg[r * (kNB + 1) + c] = (c < nb) ? v : (r == c ? 1.0 : 0.0);   // rows nb..31 (if any) ride along
    }
    for (int e = tid + nr * kNB; e < kNB * kNB; e += nt) {  // rows of Dg beyond nr (tiny last panel)
      int r = e / kNB, c = e % kNB;
      if (r >= nr) Dg[r * (kNB + 1) + c] = (r == c) ? 1.0 : 0.0;
    }
    __syncthreads();
    // (a) diagonal block: lane = row, the row lives in registers; column c is broadcast with shuffles
    if (warp == 0) {
      double row[kNB];
#pragma unroll
      for (int c = 0; c < kNB; c++) row[c] = Dg[lane * (kNB + 1) + c];
      bool bad = false;
#pragma unroll
      for (int c = 0; c < kNB; c++) {
        const double dcc = __shfl_sync(0xffffffffu, row[c], c);
        const bool live = c < nb;
        if (live && (!(dcc > 0.0) || !isfinite(dcc))) bad = true;
        const double inv = (live && dcc > 0.0) ? rsqrt(dcc) : 1.0;
        const double lrc = (lane > c) ? row[c] * inv : 0.0;
        if (lane > c) row[c] = lrc;
        if (lane == c) { row[c] = live ? dcc * inv : row[c]; if (live) invd[k0 + c] = inv; }
#pragma unroll
        for (int c2 = c + 1; c2 < kNB; c2++) {
          const double l2 = __shfl_sync(0xffffffffu, lrc, c2);   // L[c2][c]
          if (live && c2 <= lane && c2 < nb) row[c2] -= lrc * l2;
        }
      }
      if (bad) fail = 1;
#pragma unroll
      for (int c = 0; c < kNB; c++) Dg[lane * (kNB + 1) + c] = row[c];
    }
    __syncthreads();
    // (b) rows below the diagonal block: x L_d^T = a, one row per thread
    for (int r = kNB + tid; r < nr; r += nt) {
      double a[kNB];
#pragma unroll
      for (int c = 0; c < kNB; c++) a[c] = Pt[c * ldp + r];
#pragma unroll
      for (int c = 0; c < kNB; c++) {
        double s_ = a[c];
#pragma unroll
        for (int k = 0; k < c; k++) s_ -= a[k] * Dg[c * (kNB + 1) + k];
        a[c] = (c < nb) ? s_ * invd[k0 + c] : 0.0;
      }
#pragma unroll
      for (int c = 0; c < kNB; c++) Pt[c * ldp + r] = a[c];
    }
    // factored diagonal block back into the panel (rows < kNB)
    for (int e = tid; e < kNB * kNB; e += nt) {
      int r = e / kNB, c = e % kNB;
      if (r < nr && c <= r && c < nb) Pt[c * ldp + r] = Dg[r * (kNB + 1) + c];
    }
    __syncthreads();
    // write the factored panel back
    for (int e = tid; e < nr * kNB; e += nt) {
      int r = e / kNB, c = e % kNB;
      if (c < nb && r >= c) S[(size_t)(k0 + r) * ld + k0 + c] = Pt[c * ldp + r];
    }
    // (c) trailing update S[i][j] -= sum_c P[i][c] P[j][c], i >= j >= k0+nb, 4x4 register tiles
    const int t0 = nb;                  // panel-local first trailing row
    const int ntr = nr - t0;            // trailing rows (incl. rhs row)
    const int nt4 = (ntr + 3) / 4;
    const int ntri = nt4 * (nt4 + 1) / 2;
    for (int tile = tid; tile < ntri; tile += nt) {
      // triangular index -> (ti, tj), tj <= ti
      int ti = (int)((sqrt(8.0 * tile + 1.0) - 1.0) * 0.5);
      while ((ti + 1) * (ti + 2) / 2 <= tile) ti++;
      while (ti * (ti + 1) / 2 > tile) ti--;
      int tj = tile - ti * (ti + 1) / 2;
      int ri = t0 + ti * 4, rj = t0 + tj * 4;
      double a[4][4] = {};
      for (int c = 0; c < nb; c++) {
        const double *pc = Pt + c * ldp;
        double vi[4], vj[4];
#pragma unroll
        for (int q = 0; q < 4; q++) { vi[q] = (ri + q < nr) ? pc[ri + q] : 0.0; vj[q] = (rj + q < nr) ? pc[rj + q] : 0.0; }
#pragma unroll
        for (int p = 0; p < 4; p++)
#pragma unroll
          for (int q = 0; q < 4; q++) a[p][q] += vi[p] * vj[q];
      }
#pragma unroll
      for (int p = 0; p < 4; p++)
#pragma unroll
        for (int q = 0; q < 4; q++) {
          int gi = k0 + ri + p, gj = k0 + rj + q;
          if (gi < n1 && gj < n && gj <= gi) S[(size_t)gi * ld + gj] -= a[p][q];
        }
    }
    __syncthreads();
  }
  if (fail) { if (tid == 0) ctl->chol_fail = 1; return; }
  // ---- back substitution  L^T x = y, blocked from the last block
  const int nblk = (n + kNB - 1) / kNB;
  const double *y = S + (size_t)n * ld;
  for (int b = nblk - 1; b >= 0; b--) {
    const int k0 = b * kNB, nb = min(kNB, n - k0);
    // partial sums over already solved x_k, k >= k0+nb: 16 slices x 32 columns
    const int col = tid & 31, slice = tid >> 5, nslice = nt >> 5;
    double s = 0;
    if (col < nb)
      for (int k = k0 + nb + slice; k < n; k += nslice) s += S[(size_t)k * ld + k0 + col] * xs[k];
    redb[slice * 32 + col] = s;
    for (int e = tid; e < kNB * kNB; e += nt) {
      int i = e / kNB, j = e % kNB;
      Dg[i * (kNB + 1) + j] = (i < nb && j <= i) ? S[(size_t)(k0 + i) * ld + k0 + j] : 0.0;
    }
    __syncthreads();
    if (tid < 32) {
      double acc = 0;
      for (int q = 0; q < (nt >> 5); q++) acc += redb[q * 32 + tid];
      double rhs = (tid < nb) ? y[k0 + tid] - acc : 0.0;
      const double myinv = (tid < nb) ? invd[k0 + tid] : 1.0;
      // x_i = (rhs_i - sum_{j>i} L[j][i] x_j) / L[i][i], lanes hold the running right-hand sides
      double xi = 0;
      for (int i = nb - 1; i >= 0; i--) {
        double v = __shfl_sync(0xffffffffu, rhs * myinv, i);
        if (tid == i) xi = v;
        if (tid < i) rhs -= Dg[i * (kNB + 1) + tid] * v;
      }
      if (tid < nb) xs[k0 + tid] = xi;
    }
    __syncthreads();
  }
  double *gn = d.gn_c + w.offc + c0;
  for (int i = tid; i < n; i += nt) gn[i] = -xs[i];
}

// ------------------------------------------------------------------------------------------------
// Shared-memory Cholesky for reduced systems that fit one SM (n_c <= ~165: the single-drone window).
// The whole bordered matrix lives in shared memory (row-major, even leading dimension); 8-column panels:
//   (1) 8x8 diagonal block in the registers of 8 lanes: unscaled elimination whose per-column dependency chain is
//       shuffle -> reciprocal -> one DFMA, columns scaled by 1/sqrt(d) afterwards,
//   (2) TRSM of the rows below, one row per thread, against the row-scaled block (one DFMA per step on the chain),
//   (3) trailing update on the fp64 tensor cores: 8x8 output tiles, two DMMA m8n8k4 per tile, operands from a
//       transposed copy of the panel; the tile column of the next panel first, then warp 0 factors the next
//       diagonal block while the other warps update the rest.
// Then blocked back substitution, all from shared memory.  (H100's fp64 tensor-core peak is twice its DFMA peak, and
// one DMMA m8n8k4 (256 FMAs per warp) does the work of 8 DFMA per lane, so the tensor-core form wins on issue slots.)
constexpr int kCsThreads = 512;
constexpr int kCsNB = 8;
__host__ __device__ inline int chol_smem_ld(int n) { return (n + 1) & ~1; }
__host__ __device__ inline size_t chol_smem_bytes(int n) {
  size_t pr = (size_t)kCsNB * ((n + 2) & ~1), need = (size_t)n + 1 + 16 * 32;
  return ((size_t)(n + 1) * chol_smem_ld(n) + (size_t)((n + 1) & ~1) + (pr > need ? pr : need)) * 8 + 32;   // invd padded to even: P stays 16 B aligned
}
// 1/d to full double precision: fp32 MUFU seed + two Newton steps; d must be a normal positive number in float range
D2BA_DEV double fast_rcp(double d) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));   // MUFU.RCP64H: ~20 good bits, no fp32 round trip
  double e = fma(-d, r, 1.0); r = fma(r, e, r);
  e = fma(-d, r, 1.0); r = fma(r, e, r);
  e = fma(-d, r, 1.0); r = fma(r, e, r);   // third step: the seed is only guaranteed to ~2^-19, keep a safety margin
  return r;
}
// 8x8 diagonal block at (k0, k0): lanes 0..7 of one warp hold one row each in registers.  Writes L_d back, 1/L_cc
// into invd and the row-scaled block M[c][k] = L[c][k] / L[c][c] (k < c) into Ms.  Returns true on a bad pivot.
D2BA_DEV bool chol_diag8(double *A, int ld, double *invd, double *Ms, int msld, int k0, int nb, int lane) {
  double row[kCsNB];
  const int r = k0 + lane;
#pragma unroll
  for (int c = 0; c < kCsNB; c++) row[c] = (lane < nb && c <= lane) ? A[(size_t)r * ld + k0 + c] : (c == lane ? 1.0 : 0.0);
  bool bad = false;
  double dmine = 1.0;   // pivot of this lane's own column
#pragma unroll
  for (int c = 0; c < kCsNB; c++) {
    const double dcc = __shfl_sync(0xffffffffu, row[c], c);
    const bool live = c < nb;
    const bool pos = dcc > 1e-30 && dcc < 1e30;
    if (live && !pos) bad = true;
    if (lane == c) dmine = dcc;
    const double uc = row[c];   // unscaled entry of this lane in column c
    double pr[kCsNB];
#pragma unroll
    for (int c2 = c + 1; c2 < kCsNB; c2++) pr[c2] = uc * __shfl_sync(0xffffffffu, uc, c2);   // independent of the reciprocal
    const double rc = (live && pos) ? fast_rcp(dcc) : 0.0;
#pragma unroll
    for (int c2 = c + 1; c2 < kCsNB; c2++)
      if (c2 <= lane) row[c2] = fma(-pr[c2], rc, row[c2]);
  }
  // scale: L[r][c] = U[r][c] / sqrt(d_c)
  const double smine = (lane < nb && dmine > 1e-30 && dmine < 1e30) ? fast_rsqrt(dmine) : 1.0;
  double sc[kCsNB];
#pragma unroll
  for (int c = 0; c < kCsNB; c++) sc[c] = __shfl_sync(0xffffffffu, smine, c);
  if (lane < nb) {
    invd[k0 + lane] = smine;
#pragma unroll
    for (int c = 0; c < kCsNB; c++) {
      const double l = row[c] * sc[c];
      if (c <= lane) A[(size_t)r * ld + k0 + c] = l;
      Ms[lane * msld + c] = (c < lane) ? l * smine : 0.0;
    }
  } else if (lane < kCsNB) {
#pragma unroll
    for (int c = 0; c < kCsNB; c++) Ms[lane * msld + c] = 0.0;
  }
  return bad;
}

// C(8x8 at rows gi0.., cols gj0..) -= P^T P over the 8 panel columns; rows >= n1 and the strict upper part of a
// diagonal tile are not stored.  pmax = last readable index of a row of the panel copy.
D2BA_DEV void chol_tile8(double *A, int ld, const double *P, int ldp, int gi0, int gj0, int ri, int rj, int pmax, int n1, bool diag_tile, int lane) {
  const int q = lane & 3, g = lane >> 2;
  const int ia = min(ri + g, pmax), ib = min(rj + g, pmax);
  const double a0 = -P[q * ldp + ia], a1 = -P[(q + 4) * ldp + ia];
  const double b0 = P[q * ldp + ib], b1 = P[(q + 4) * ldp + ib];
  const int gi = gi0 + g, gj = gj0 + 2 * q;
  const bool rowok = gi < n1;
  double2 *dst = reinterpret_cast<double2 *>(A + (size_t)gi * ld + gj);
  double2 c = rowok ? *dst : make_double2(0.0, 0.0);
  dmma(c.x, c.y, a0, b0);
  dmma(c.x, c.y, a1, b1);
  if (rowok) {
    if (!diag_tile && gj0 + 8 <= n1 - 1) *dst = c;   // interior tile: all 8 columns are matrix columns below the diagonal
    else {
      if (gj <= gi && gj < n1 - 1) A[(size_t)gi * ld + gj] = c.x;
      if (gj + 1 <= gi && gj + 1 < n1 - 1) A[(size_t)gi * ld + gj + 1] = c.y;
    }
  }
}

__global__ void __launch_bounds__(kCsThreads) k_chol_smem(Dev d) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  if (!w.chol_smem) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse || ctl->chol_fail) return;
  extern __shared__ __align__(16) double sm[];
  // after the speed-bias elimination (k_sb_elim + Schur) only the landmark-coupled part is left: S rows 0..n_lc (rhs)
  // ... and after the leaf elimination only the hub [hub0, n_lc) of it
  const bool reduced = w.sb_elim != 0 || w.n_leaf > 0;
  const int c0 = reduced ? w.hub0 : 0;
  const int n = reduced ? w.n_hub : w.n_c, n1 = n + 1, ld = chol_smem_ld(n), ldg = w.ldh, ldp = (n + 2) & ~1;
  double *A = sm;                         // n1 x ld
  double *invd = A + (size_t)n1 * ld;     // n (padded to even)
  double *P = invd + ((n + 1) & ~1);      // kCsNB x ldp transposed panel; later xs / partial sums
  const double *S = d.S + w.offH + (size_t)c0 * ldg + c0;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  __shared__ int fail;
  // row-scaled diagonal block for the TRSM: parked in the (never touched) upper-right corner of A, or behind the panel
  // copy when the matrix is too small to have one
  double *Ms = n >= 32 ? A + (ld - kCsNB) : P + (size_t)kCsNB * ldp;
  const int msld = n >= 32 ? ld : kCsNB;
  if (tid == 0) fail = 0;
#ifdef D2BA_CHOL_TIMING
  long long tk[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; long long tq = clock64();
#define TLAP(k) do { long long t_ = clock64(); tk[k] += t_ - tq; tq = t_; } while (0)
#else
#define TLAP(k) do { } while (0)
#endif
  // load the lower triangle (+ rhs row) with one TMA bulk copy per row, all in flight at once.  Rows of the
  // landmark-coupled part come from the Schur kernel's S; when that was the one-CTA kernel the speed-bias rows are
  // taken from Hcc directly (+ mu D^2 on the diagonal, added below) and their share of u^T H u is accumulated here.
  {
    __shared__ __align__(8) unsigned long long bar;
    const int nlc = w.n_lc, cur = ctl->cur;
    const bool direct = !reduced && w.schur_small != 0;
    const double *H = d.Hcc[cur] + w.offH, *gcv = d.gc[cur] + w.offc, *ucv = d.uc + w.offc, *D2v = d.D2c + w.offc;
    const int nbulk = direct ? n : n1;               // rows copied by TMA; the rhs row of the direct case is stitched by hand
    if (tid == 0) { mbar_init(&bar, 1); mbar_fence_init(); }
    __syncthreads();
    if (warp == 0) {
      if (lane == 0) {
        unsigned total = 0;
        for (int r = 0; r < nbulk; r++) total += (unsigned)(((min(r, n - 1) + 2) & ~1) * 8);
        mbar_expect_tx(&bar, total);
      }
      __syncwarp();
      for (int r = lane; r < nbulk; r += 32) {
        const double *src = ((direct && r >= nlc) ? H : S) + (size_t)r * ldg;
        bulk_g2s(A + (size_t)r * ld, src, (unsigned)(((min(r, n - 1) + 2) & ~1) * 8), &bar);
      }
    }
    if (direct) {
      const double *src = S + (size_t)n * ldg;
      double *dst = A + (size_t)n * ld;
      for (int c = tid; c < n; c += nt) dst[c] = c < nlc ? src[c] : gcv[c];
    }
    mbar_wait(&bar, 0);
    if (direct) {
      const double mu = ctl->mu;
      double uhu = 0.0;
      for (int r = nlc + warp; r < n; r += nwarp) {
        const double *row = A + (size_t)r * ld;
        const double ur = ucv[r];
        double acc = 0.0;
        for (int c = lane; c < r; c += 32) acc += row[c] * ucv[c];
        uhu += 2.0 * acc * ur;
        if (lane == 0) { const double v = row[r]; uhu += v * ur * ur; A[(size_t)r * ld + r] = v + mu * D2v[r]; }
      }
      uhu = warp_sum(uhu);
      if (lane == 0 && uhu != 0.0) atomicAdd(&ctl->uHu_cam, uhu);
    }
  }
  __syncthreads();
  TLAP(0);
  if (warp == 0) { if (chol_diag8(A, ld, invd, Ms, msld, 0, min(kCsNB, n), lane)) fail = 1; }
  __syncthreads();
  TLAP(1);
  for (int k0 = 0; k0 < n; k0 += kCsNB) {
    const int nb = min(kCsNB, n - k0), nxt = k0 + nb;
    // (2) rows below the (already factored) diagonal block: a L_d^T = x; results also into the transposed copy P[c][r - k0]
    for (int r = nxt + tid; r < n1; r += nt) {
      double a[kCsNB];
      double *ar = A + (size_t)r * ld + k0;
#pragma unroll
      for (int c = 0; c < kCsNB; c++) a[c] = (c < nb) ? ar[c] * invd[k0 + c] : 0.0;
#pragma unroll
      for (int c = 1; c < kCsNB; c++) {
        double s_ = a[c];
#pragma unroll
        for (int k = 0; k < c; k++) s_ = fma(-a[k], Ms[c * msld + k], s_);
        a[c] = s_;
      }
#pragma unroll
      for (int c = 0; c < kCsNB; c++) { if (c < nb) ar[c] = a[c]; P[c * ldp + (r - k0)] = a[c]; }
    }
    TLAP(2);
    __syncthreads();
    TLAP(3);
    if (nxt >= n) break;
    const int nb2 = min(kCsNB, n - nxt);
    const int pmax = n - k0;                           // P rows hold indices [nb, n1 - 1 - k0]
    const int T8 = (n1 - nxt + 7) >> 3;                // 8-row tiles of the trailing matrix (rows / cols from nxt)
    // (3a) look-ahead: the tile column of the next panel, all warps
    for (int ti = warp; ti < T8; ti += nwarp)
      chol_tile8(A, ld, P, ldp, nxt + 8 * ti, nxt, nb + 8 * ti, nb, pmax, n1, ti == 0, lane);
    __syncthreads();
    TLAP(4);
    // (3b) warp 0 factors the next diagonal block while the other warps update the rest of the trailing matrix
    if (warp == 0) {
      if (chol_diag8(A, ld, invd, Ms, msld, nxt, nb2, lane)) fail = 1;
    } else {
      // warps 4, 8, 12 share warp 0's scheduler / fp64 pipe: they sit this phase out once the trailing matrix is
      // small enough that the diagonal block (a pure latency chain) is the longer of the two jobs
      const int T = T8 - 1;                            // tiles per side without the first tile column
      const int ntile = T * (T + 1) / 2;
      const bool spare = ntile <= 140;
      if (!(spare && (warp & 3) == 0)) {
        const int wslot = spare ? (warp - 1 - (warp >> 2)) : (warp - 1), nslot = spare ? nwarp - (nwarp >> 2) : nwarp - 1;
        int ti = 0, tj = wslot;                        // tile (ti, tj) of the lower triangle, row-major enumeration
        while (tj > ti) { tj -= ti + 1; ti++; }
        while (ti < T) {
          chol_tile8(A, ld, P, ldp, nxt + 8 * (ti + 1), nxt + 8 * (tj + 1), nb + 8 * (ti + 1), nb + 8 * (tj + 1), pmax, n1, ti == tj, lane);
          tj += nslot;
          while (tj > ti) { tj -= ti + 1; ti++; }
        }
      }
    }
    TLAP(5);
    __syncthreads();
    TLAP(6);
  }
  if (fail) { if (tid == 0) ctl->chol_fail = 1; return; }
  // ---- back substitution L^T x = y (y = row n), 32-column blocks from the end
  double *xs = P;                 // n
  double *redb = P + n + 1;       // 16 x 32
  const double *y = A + (size_t)n * ld;
  const int nblk = (n + 31) / 32;
  for (int b = nblk - 1; b >= 0; b--) {
    const int k0 = b * 32, nb = min(32, n - k0);
    const int col = tid & 31, slice = tid >> 5, nslice = nt >> 5;
    double s_ = 0;
    if (col < nb)
      for (int k = k0 + nb + slice; k < n; k += nslice) s_ += A[(size_t)k * ld + k0 + col] * xs[k];
    redb[slice * 32 + col] = s_;
    TLAP(7);
    __syncthreads();
    if (tid < 32) {
      double acc = 0;
#pragma unroll 4
      for (int q = 0; q < nslice; q++) acc += redb[q * 32 + tid];
      double rhs = (tid < nb) ? y[k0 + tid] - acc : 0.0;
      const double myinv = (tid < nb) ? invd[k0 + tid] : 1.0;
      double lcol[32];   // L[k0 + i][k0 + tid] for i > tid: the triangular solve below then runs register / shuffle only
#pragma unroll
      for (int i = 0; i < 32; i++) lcol[i] = (i < nb && tid < i) ? A[(size_t)(k0 + i) * ld + k0 + tid] : 0.0;
      double xi = 0;
#pragma unroll
      for (int i = 31; i >= 0; i--) {
        const double v = __shfl_sync(0xffffffffu, rhs * myinv, i);
        if (tid == i) xi = v;
        rhs -= lcol[i] * v;
      }
      if (tid < nb) xs[k0 + tid] = xi;
    }
    TLAP(8);
    __syncthreads();
  }
  double *gn = d.gn_c + w.offc + c0;
  for (int i = tid; i < n; i += nt) gn[i] = -xs[i];
#ifdef D2BA_CHOL_TIMING
  TLAP(9);
  if (wi == 0 && (tid == 0 || tid == 32 || tid == 480))
    printf("chol timing tid %d n %d: load %lld diag0 %lld trsm %lld trsm_bar %lld look+bar %lld work3b %lld bar3b %lld back_partial %lld back_tri %lld tail %lld\n", tid, n,
           tk[0], tk[1], tk[2], tk[3], tk[4], tk[5], tk[6], tk[7], tk[8], tk[9]);
#endif
}

// ------------------------------------------------------------------------------------------------
// Speed-bias elimination (arrow structure of the visual-inertial reduced system).
// Columns are ordered [poses / extrinsics / td | speed-bias blocks]; the speed-bias block S_ss is block tridiagonal
// (IMU factors couple consecutive frames only) while its coupling B to the landmark-coupled part is dense.  Instead of
// one dense Cholesky of all n_c columns (a chain of n_c dependent column steps on a matrix that fills one SM's shared
// memory), the speed-bias blocks are eliminated first with a block-bidiagonal Cholesky
//     L_kk L_kk^T = D_k - E'_{k-1} E'_{k-1}^T,   E'_k = E_k L_kk^-T,   Y_k = L_kk^-1 (B_k - E'_{k-1} Y_{k-1})
// ([B | g_s] carries the right-hand side as its last column).  The rows Y are appended to the scaled landmark rows Wt,
// so the Schur kernel that runs next forms  S_pp + mu D^2 - Wt^T Wt - Y^T Y  and  g_p - Wt^T g~ - Y^T z_s  in one
// tensor-core SYRK: the dense part shrinks to n_lc x n_lc, which k_chol_smem factors with several windows per SM (or
// k_chol for multi-agent windows), and k_sb_back recovers the speed-bias step from
//     L_kk^T x_k = z_k - Y_k x_p - E'_k^T x_{k+1}.
// Same normal equations, another (equally stable) elimination order than the reference's dense LLT.
// (constants and the kernel follow chol_block9)
// Cholesky of one 9x9 block held in shared memory (row stride 9), lanes 0..8 own one row each.  Unscaled elimination
// with the reciprocal chain of chol_diag8; L overwrites the lower part, 1/L_ii goes to invd.  Returns true on a bad pivot.
D2BA_DEV bool chol_block9(double *Dk, double *invd, int lane) {
  constexpr int NB = 9;
  double row[NB];
#pragma unroll
  for (int c = 0; c < NB; c++) row[c] = (lane < NB && c <= lane) ? Dk[lane * NB + c] : 0.0;
  bool bad = false;
  double dmine = 1.0;
#pragma unroll
  for (int c = 0; c < NB; c++) {
    const double dcc = __shfl_sync(0xffffffffu, row[c], c);
    const bool pos = dcc > 1e-30 && dcc < 1e30;
    if (!pos) bad = true;
    if (lane == c) dmine = dcc;
    const double uc = row[c];
    double pr[NB];
#pragma unroll
    for (int c2 = c + 1; c2 < NB; c2++) pr[c2] = uc * __shfl_sync(0xffffffffu, uc, c2);
    const double rc = pos ? fast_rcp(dcc) : 0.0;
#pragma unroll
    for (int c2 = c + 1; c2 < NB; c2++)
      if (c2 <= lane) row[c2] = fma(-pr[c2], rc, row[c2]);
  }
  const double smine = (lane < NB && dmine > 1e-30 && dmine < 1e30) ? fast_rsqrt(dmine) : 1.0;
  double sc[NB];
#pragma unroll
  for (int c = 0; c < NB; c++) sc[c] = __shfl_sync(0xffffffffu, smine, c);
  if (lane < NB) {
    invd[lane] = smine;
#pragma unroll
    for (int c = 0; c < NB; c++) if (c <= lane) Dk[lane * NB + c] = row[c] * sc[c];
  }
  return bad;
}

constexpr int kSeThreads = 128;    // warp 0: D / E chain, warps 1..3: Y rows
constexpr int kSeMaxBlocks = 32;   // speed-bias blocks per window (mbarrier table)
constexpr int kSeSlotRows = 9;
__host__ __device__ inline size_t sbe_smem_bytes(int ldw, int n_c, int nb) {
  return ((size_t)3 * kSeSlotRows * ldw + (size_t)nb * 2 * 81 + (size_t)nb * 9 + (size_t)n_c + (size_t)9 * nb + 16) * 8;
}

__global__ void __launch_bounds__(kSeThreads, 4) k_sb_elim(Dev d) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  if (!w.sb_elim) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse || ctl->chol_fail) return;
  extern __shared__ __align__(16) double sm[];
  const int nlc = w.n_lc, nb = w.n_sbe, n = w.n_c, ld = w.ldh, cur = ctl->cur;
  // the speed-bias blocks couple (IMU factors, prior) only to hub columns [hub0, n_lc): the B rows are that wide
  const int c0 = w.hub0, nh = nlc - c0, ldgw = w.ldw;
  const int ldys = (nh + 1 + 7) & ~7, ncol = nh + 1, slot_sz = kSeSlotRows * ldys;   // ring rows: multiple of 8, >= n_hub + 1
  double *Yr = sm;                                  // ring of 3 slots x 9 rows x ldw: [B_k | g_k] -> Y_k
  double *Dk = Yr + (size_t)3 * slot_sz;            // nb x 81 : D_k -> L_kk
  double *Ek = Dk + (size_t)nb * 81;                // nb x 81 : E_k (rows: block k+1, cols: block k) -> E'_k
  double *invd = Ek + (size_t)nb * 81;              // nb x 9
  double *us = invd + (size_t)nb * 9;               // n : u = g / D^2 of the accepted linearisation
  double *gs = us + n;                              // 9 nb : speed-bias part of the gradient
  const double *H = d.Hcc[cur] + w.offH, *gcv = d.gc[cur] + w.offc, *ucv = d.uc + w.offc, *D2v = d.D2c + w.offc;
  double *Yg = d.Wt + w.offW + (size_t)w.nl * w.ldw;   // the eliminated rows follow the landmark rows of Wt directly
  const double mu = ctl->mu;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  __shared__ int fail;
  __shared__ __align__(8) unsigned long long bar_B[kSeMaxBlocks], bar_L[kSeMaxBlocks], bar_E[kSeMaxBlocks];
  if (tid == 0) {
    fail = 0;
    for (int k = 0; k < nb; k++) { mbar_init(&bar_B[k], 1); mbar_init(&bar_L[k], 1); mbar_init(&bar_E[k], 1); }
    mbar_fence_init();
  }
  __syncthreads();
  // B rows of a block: one TMA bulk copy per row into ring slot k % 3 (issued by one follower lane, two blocks ahead)
  const unsigned row_bytes = (unsigned)(((nh + 1) & ~1) * 8);   // hub0 is a multiple of 6 (even): 16-byte aligned source
  auto issue_rows = [&](int k) {
    mbar_expect_tx(&bar_B[k], 9u * row_bytes);
    double *dst = Yr + (size_t)(k % 3) * slot_sz;
    for (int i = 0; i < 9; i++) bulk_g2s(dst + (size_t)i * ldys, H + (size_t)(nlc + 9 * k + i) * ld + c0, row_bytes, &bar_B[k]);
  };
  if (tid == 32) { issue_rows(0); if (nb > 1) issue_rows(1); }
  // ---- the 9x9 blocks, u, g_s (8-byte cp.async: everything in flight at once); the blocks' share of u^T H u; mu D^2
  for (int e = tid; e < n; e += nt) cp_async8(us + e, ucv + e);
  for (int e = tid; e < 9 * nb * 18; e += nt) {
    const int r = e / 18, q = e - 18 * r, k = r / 9, i = r - 9 * k, j = q % 9;
    const double *hr = H + (size_t)(nlc + r) * ld;
    if (q < 9) { if (k > 0) cp_async8(Ek + (size_t)(k - 1) * 81 + i * 9 + j, hr + nlc + 9 * (k - 1) + j); }
    else cp_async8(Dk + (size_t)k * 81 + i * 9 + j, hr + nlc + 9 * k + j);
  }
  for (int e = tid; e < 9 * nb; e += nt) cp_async8(gs + e, gcv + nlc + e);
  cp_async_wait_all();
  __syncthreads();
  double uhu = 0.0;
  for (int e = tid; e < 9 * nb * 18; e += nt) {
    const int r = e / 18, q = e - 18 * r, k = r / 9, i = r - 9 * k, j = q % 9;
    const double ur = us[nlc + r];
    if (q < 9) { if (k > 0) uhu += 2.0 * ur * Ek[(size_t)(k - 1) * 81 + i * 9 + j] * us[nlc + 9 * (k - 1) + j]; }
    else if (j < i) uhu += 2.0 * ur * Dk[(size_t)k * 81 + i * 9 + j] * us[nlc + 9 * k + j];
    else if (j == i) uhu += Dk[(size_t)k * 81 + i * 9 + i] * ur * ur;
  }
  __syncthreads();
  for (int e = tid; e < 9 * nb; e += nt) Dk[(size_t)(e / 9) * 81 + (e % 9) * 10] += mu * D2v[nlc + e];
  __syncthreads();
  if (warp == 0) {
    // ---- the D / E chain: chol(D_k) -> E'_k = E_k L_kk^-T -> D_{k+1} -= E'_k E'_k^T, each block published by an mbarrier
    for (int k = 0; k < nb; k++) {
      double *Lk = Dk + (size_t)k * 81, *iv = invd + k * 9;
      if (chol_block9(Lk, iv, lane)) fail = 1;
      __threadfence_block();
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_L[k]);
      if (k + 1 < nb) {
        double *Ep = Ek + (size_t)k * 81;
        if (lane < 9) {
          double *er = Ep + lane * 9;
          double a[9];
#pragma unroll
          for (int c = 0; c < 9; c++) a[c] = er[c];
#pragma unroll
          for (int c = 0; c < 9; c++) {
            double s_ = a[c];
#pragma unroll
            for (int j = 0; j < c; j++) s_ = fma(-a[j], Lk[c * 9 + j], s_);
            a[c] = s_ * iv[c];
          }
#pragma unroll
          for (int c = 0; c < 9; c++) er[c] = a[c];
        }
        __syncwarp();
        double *Dn = Dk + (size_t)(k + 1) * 81;
        for (int e = lane; e < 81; e += 32) {
          const int i = e / 9, j = e - 9 * i;
          double s_ = 0.0;
#pragma unroll
          for (int m = 0; m < 9; m++) s_ += Ep[i * 9 + m] * Ep[j * 9 + m];
          Dn[e] -= s_;
        }
        __threadfence_block();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bar_E[k]);
      }
    }
  } else {
    // ---- followers: per block  Y_k = L_kk^-1 ([B_k | g_k] - E'_{k-1} Y_{k-1}), one column per thread in registers;
    //      the rows go to Wt (behind the landmark rows), so the Schur kernel that follows subtracts Y^T Y together with
    //      the landmark terms and k_sb_back finds them there
    const int t1 = tid - 32, n1t = nt - 32;
    for (int k = 0; k < nb; k++) {
      double *Yk = Yr + (size_t)(k % 3) * slot_sz;
      const double *Yp = Yr + (size_t)((k + 2) % 3) * slot_sz;   // slot of block k-1
      mbar_wait(&bar_B[k], 0);
      if (k > 0) mbar_wait(&bar_E[k - 1], 0);
      mbar_wait(&bar_L[k], 0);
      const double *Lk = Dk + (size_t)k * 81, *iv = invd + k * 9, *Ep = Ek + (size_t)(k > 0 ? k - 1 : 0) * 81;
      for (int c = t1; c < ldys; c += n1t) {
        double y[9];
        if (c < nh) {
          double ub = 0.0;
#pragma unroll
          for (int i = 0; i < 9; i++) { y[i] = Yk[(size_t)i * ldys + c]; ub += y[i] * us[nlc + 9 * k + i]; }
          uhu += 2.0 * ub * us[c0 + c];
        } else {
#pragma unroll
          for (int i = 0; i < 9; i++) y[i] = c == nh ? gs[9 * k + i] : 0.0;
        }
        if (c < ncol) {
          if (k > 0) {
            double yp[9];
#pragma unroll
            for (int m = 0; m < 9; m++) yp[m] = Yp[(size_t)m * ldys + c];
#pragma unroll
            for (int i = 0; i < 9; i++)
#pragma unroll
              for (int m = 0; m < 9; m++) y[i] = fma(-Ep[i * 9 + m], yp[m], y[i]);
          }
#pragma unroll
          for (int i = 0; i < 9; i++) {
            double s_ = y[i];
#pragma unroll
            for (int j = 0; j < i; j++) s_ = fma(-Lk[i * 9 + j], y[j], s_);
            y[i] = s_ * iv[i];
          }
        }
#pragma unroll
        for (int i = 0; i < 9; i++) { Yk[(size_t)i * ldys + c] = y[i]; if (c < ncol) Yg[(size_t)(9 * k + i) * ldgw + c0 + c] = y[i]; }
      }
      asm volatile("bar.sync 1, %0;" ::"r"(n1t) : "memory");   // slot (k+2) % 3 == slot of block k-1 is dead now
      if (t1 == 0 && k + 2 < nb) { fence_proxy_async(); issue_rows(k + 2); }
    }
  }
  uhu = warp_sum(uhu);
  if (lane == 0 && uhu != 0.0) atomicAdd(&ctl->uHu_cam, uhu);
  __syncthreads();
  if (fail) { if (tid == 0) ctl->chol_fail = 1; return; }
  double *LE = d.sbLE + w.offLE;
  for (int e = tid; e < nb * 81; e += nt) { LE[e] = Dk[e]; LE[(size_t)nb * 81 + e] = Ek[e]; }
  for (int e = tid; e < nb * 9; e += nt) LE[(size_t)nb * 162 + e] = invd[e];
}

// Speed-bias part of the Gauss-Newton step: L_kk^T x_k = z_k - Y_k x_p - E'_k^T x_{k+1}, blocks from the last to the
// first.  One CTA per window: all warps form v = Y x_p (coalesced, many loads in flight) and stage the small blocks,
// warp 0 then runs the short recursion out of shared memory.
constexpr int kSbBackThreads = 256;
__host__ __device__ inline size_t sb_back_smem_bytes(int nlc, int nb) { return (size_t)(((nlc + 31) & ~31) + 9 * nb + 171 * nb) * 8; }
__global__ void __launch_bounds__(kSbBackThreads) k_sb_back(Dev d) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  if (!w.sb_elim) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done || ctl->reuse || ctl->chol_fail) return;
  extern __shared__ double sm[];
  const int c0 = w.hub0, nh = w.n_lc - c0, nlc = w.n_lc, nb = w.n_sbe, ldy = w.ldw;   // Y lives in the hub columns [hub0, n_lc] of its rows
  double *xp = sm;                       // n_hub (padded to 32)
  double *rhs = sm + ((nh + 31) & ~31);  // 9 nb : z - Y x_p
  double *LE = rhs + 9 * nb;             // nb x 171
  const double *Yg = d.Wt + w.offW + (size_t)w.nl * w.ldw, *LEg = d.sbLE + w.offLE;
  double *gn = d.gn_c + w.offc;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int c = tid; c < nh; c += nt) xp[c] = -gn[c0 + c];
  for (int e = tid; e < nb * 171; e += nt) cp_async8(LE + e, LEg + e);   // needed only by the recursion: lands during the products
  __syncthreads();
  for (int r0 = warp * 4; r0 < 9 * nb; r0 += nwarp * 4) {
    double s_[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int q = 0; q < 4; q++) {
      if (r0 + q >= 9 * nb) break;
      const double *yr = Yg + (size_t)(r0 + q) * ldy + c0;
      for (int c = lane; c < nh; c += 32) s_[q] += yr[c] * xp[c];
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const double t = warp_sum(s_[q]);
      if (lane == 0 && r0 + q < 9 * nb) rhs[r0 + q] = Yg[(size_t)(r0 + q) * ldy + nlc] - t;
    }
  }
  cp_async_wait_all();
  __syncthreads();
  if (warp != 0) return;
  const double *Lg = LE, *Eg = LE + (size_t)nb * 81, *ivg = LE + (size_t)nb * 162;
  double xn = 0.0;   // lane i < 9 holds x_{k+1}[i]
  for (int k = nb - 1; k >= 0; k--) {
    double t = lane < 9 ? rhs[9 * k + lane] : 0.0;
    if (k + 1 < nb) {   // - E'_k^T x_{k+1}: entry i = sum_m E'_k[m][i] x_{k+1}[m]
      const double *E = Eg + (size_t)k * 81;
#pragma unroll
      for (int m = 0; m < 9; m++) {
        const double xm = __shfl_sync(0xffffffffu, xn, m);
        if (lane < 9) t -= E[m * 9 + lane] * xm;
      }
    }
    // L_kk^T x = t, from the last entry up
    const double *L = Lg + (size_t)k * 81;
    const double myinv = lane < 9 ? ivg[k * 9 + lane] : 1.0;
    double lcol[9];
#pragma unroll
    for (int i = 0; i < 9; i++) lcol[i] = lane < i ? L[i * 9 + lane] : 0.0;
    double x = 0.0;
#pragma unroll
    for (int i = 8; i >= 0; i--) {
      const double v = __shfl_sync(0xffffffffu, t * myinv, i);
      if (lane == i) x = v;
      t -= lcol[i] * v;
    }
    xn = x;
    if (lane < 9) gn[nlc + 9 * k + lane] = -x;
  }
}

// ------------------------------------------------------------------------------------------------
// Leaf elimination (multi-agent windows).  A leaf = the pose blocks of one remote drone: through the landmarks they couple
// only to themselves and to the hub (own frames / extrinsics / td), never to another leaf, so the pose part of the reduced
// system is an arrow:  [S_11 . . B_1^T; . S_22 . B_2^T; ...; B_1 B_2 ... S_hh].  One CTA per (window, leaf) factors
// S_bb = L L^T in shared memory (8-column panels: chol_diag8 on the diagonal block, one-row-per-thread TRSM, fp64
// tensor-core trailing update) with the hub rows [B_b ; g_b^T] riding along as extra rows, which turns them into
// Y_b^T = [B_b ; g_b^T] L^-T.  The rows Y_b go behind the landmark / speed-bias rows of Wt, so the hub tiles of the Schur
// kernel (which run next) subtract Y_b^T Y_b together with the landmark terms; k_leaf_back recovers the leaf step from
// L^T x_b = z_b - Y_b x_hub.  The dense Cholesky shrinks from 6 x (all poses) to the hub (66 columns for an 11-frame window).
#ifndef D2BA_LEAF_THREADS
#define D2BA_LEAF_THREADS 256
#endif
constexpr int kLeafThreads = D2BA_LEAF_THREADS;
constexpr int kLeafMaxCols = 96;
constexpr int kLeafLmChunk = 16;   // landmarks whose coupling rows are staged at a time (a multiple of the MMA k = 4)
__host__ __device__ inline int leaf_lda(int n) { return n | 1; }   // odd: the one-row-per-thread TRSM walks the rows without bank conflicts (all accesses are scalar)
__host__ __device__ inline size_t leaf_elim_smem_bytes(int n, int nh) {
  const int n1 = n + nh + 1;
  return ((size_t)n1 * leaf_lda(n) + (size_t)((n + 1) & ~1) + (size_t)kCsNB * ((n1 + 1) & ~1) + 64 + (size_t)kLeafLmChunk * n1 + 8) * 8;
}
// C(8x8 at rows gi0.., cols gj0..) -= P^T P over the 8 panel columns; rows of the leaf block (gi < n) keep the lower
// triangle only, the extra rows (gi >= n) all n columns
D2BA_DEV void leaf_tile8(double *A, int ld, const double *P, int ldp, int gi0, int gj0, int ri, int rj, int pmax, int n1, int n, int lane) {
  const int q = lane & 3, g = lane >> 2;
  const int ia = min(ri + g, pmax), ib = min(rj + g, pmax);
  const double a0 = -P[q * ldp + ia], a1 = -P[(q + 4) * ldp + ia];
  const double b0 = P[q * ldp + ib], b1 = P[(q + 4) * ldp + ib];
  const int gi = gi0 + g, gj = gj0 + 2 * q;
  const bool rowok = gi < n1 && gj < n;
  double2 c = make_double2(0.0, 0.0);
  if (rowok) { c.x = A[(size_t)gi * ld + gj]; if (gj + 1 < n) c.y = A[(size_t)gi * ld + gj + 1]; }
  dmma(c.x, c.y, a0, b0);
  dmma(c.x, c.y, a1, b1);
  if (rowok) {
    const int lim = gi < n ? gi : n - 1;   // last column of this row that is stored
    if (gj <= lim) A[(size_t)gi * ld + gj] = c.x;
    if (gj + 1 <= lim) A[(size_t)gi * ld + gj + 1] = c.y;
  }
}

// C(8x8 at rows gi0.., cols gj0..) -= W^T W over nq4 staged landmark rows (W: [landmark][n1 columns], zero padded to a
// multiple of 4 rows); same storage rule as leaf_tile8
D2BA_DEV void leaf_rank8(double *A, int ld, const double *W, int ldw, int gi0, int gj0, int nq4, int n1, int n, int lane) {
  const int q = lane & 3, g = lane >> 2;
  const int ia = min(gi0 + g, n1 - 1), ib = min(gj0 + g, n1 - 1);
  const int gi = gi0 + g, gj = gj0 + 2 * q;
  const bool rowok = gi < n1 && gj < n;
  double2 c = make_double2(0.0, 0.0);
  if (rowok) { c.x = A[(size_t)gi * ld + gj]; if (gj + 1 < n) c.y = A[(size_t)gi * ld + gj + 1]; }
  for (int ks = 0; ks < nq4; ks += 4) dmma(c.x, c.y, -W[(size_t)(ks + q) * ldw + ia], W[(size_t)(ks + q) * ldw + ib]);
  if (rowok) {
    const int lim = gi < n ? gi : n - 1;
    if (gj <= lim) A[(size_t)gi * ld + gj] = c.x;
    if (gj + 1 <= lim) A[(size_t)gi * ld + gj + 1] = c.y;
  }
}

#if D2BA_LEAF_THREADS > 256
__global__ void __launch_bounds__(kLeafThreads, 2) k_leaf_elim(Dev d) {
#else
__global__ void __launch_bounds__(kLeafThreads) k_leaf_elim(Dev d) {
#endif
  const Leaf lf = d.leaf[blockIdx.x];
  const WinDesc &w = d.win[lf.win];
  Ctl *ctl = d.ctl + lf.win;
  if (ctl->done || ctl->reuse || ctl->chol_fail) return;
  extern __shared__ __align__(16) double sm[];
  const int n = lf.n, nh = w.n_hub, n1 = n + nh + 1, lda = leaf_lda(n), ldp = (n1 + 1) & ~1, ldg = w.ldh, cur = ctl->cur;
  double *A = sm;                                   // n1 x lda: leaf block (lower), then the hub rows and the rhs row
  double *invd = A + (size_t)n1 * lda;              // n (padded to even)
  double *P = invd + ((n + 1) & ~1);                // kCsNB x ldp: transposed panel
  double *Ms = P + (size_t)kCsNB * ldp;             // 8 x 8 row-scaled diagonal block
  double *Wl = Ms + 64;                             // kLeafLmChunk x n1: coupling rows of a chunk of this leaf's landmarks
  const double *H = d.Hcc[cur] + w.offH, *gcv = d.gc[cur] + w.offc, *ucv = d.uc + w.offc, *D2v = d.D2c + w.offc;
  const double mu = ctl->mu;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  __shared__ int fail;
  if (tid == 0) fail = 0;
  // ---- this leaf's part of the reduced system, formed here:  [H_bb ; H_hub,b ; g_b^T] - sum over its landmarks of
  //      [w_l,b ; w_l,hub ; g~_l]^T w_l,b  (the leaf's landmarks touch no other leaf).  Asynchronous 8-byte copies keep the
  //      whole block in flight at once; the upper triangle of the leaf block is never read.
  for (int e = tid; e < n1 * n; e += nt) {
    const int r = e / n, c = e - r * n;
    double *dst = A + (size_t)r * lda + c;
    if (r < n) { if (c <= r) cp_async8(dst, H + (size_t)(lf.col0 + r) * ldg + lf.col0 + c); }
    else if (r < n + nh) cp_async8(dst, H + (size_t)(w.hub0 + r - n) * ldg + lf.col0 + c);
    else cp_async8(dst, gcv + lf.col0 + c);
  }
  cp_async_wait_all();
  __syncthreads();
  {   // the block's share of u^T Hcc u (lower entries, off-diagonal twice), then mu D^2 on the diagonal
    double *us = Wl;   // u of the leaf columns, then of the hub columns (the staging area is free until the rank updates)
    for (int e = tid; e < n + nh; e += nt) us[e] = e < n ? ucv[lf.col0 + e] : ucv[w.hub0 + e - n];
    __syncthreads();
    double uhu = 0.0;
    for (int e = tid; e < (n + nh) * n; e += nt) {
      const int r = e / n, c = e - r * n;
      if (r < n && c > r) continue;
      uhu += ((r < n && c == r) ? 1.0 : 2.0) * A[(size_t)r * lda + c] * us[r] * us[c];
    }
    uhu = warp_sum(uhu);
    if (lane == 0 && uhu != 0.0) atomicAdd(&ctl->uHu_cam, uhu);
    __syncthreads();
    for (int i = tid; i < n; i += nt) A[(size_t)i * lda + i] += mu * D2v[lf.col0 + i];
  }
  const double *Wt = d.Wt + w.offW;
  const int *lml = d.leaf_lm + lf.lm_begin;
  for (int l0 = 0; l0 < lf.lm_count; l0 += kLeafLmChunk) {
    const int nq = min(kLeafLmChunk, lf.lm_count - l0);
    __syncthreads();
    const int nq4 = (nq + 3) & ~3;
    for (int e = tid; e < nq4 * n1; e += nt) {
      const int q = e / n1, c = e - q * n1;
      if (q < nq) {
        const double *row = Wt + (size_t)lml[l0 + q] * w.ldw;
        cp_async8(Wl + (size_t)q * n1 + c, c < n ? row + lf.col0 + c : row + w.hub0 + (c - n));
      } else Wl[(size_t)q * n1 + c] = 0.0;
    }
    cp_async_wait_all();
    __syncthreads();
    // fp64 tensor-core rank update over the 8x8 tiles of the lower trapezoid: row tile ti has min(ti + 1, Tc0) column tiles;
    // the warps walk the tile list with stride nwarp (no division)
    const int Tr0 = (n1 + 7) >> 3, Tc0 = (n + 7) >> 3;
    for (int ti = 0, tj = warp;; ) {
      while (ti < Tr0 && tj >= min(ti + 1, Tc0)) { tj -= min(ti + 1, Tc0); ti++; }
      if (ti >= Tr0) break;
      leaf_rank8(A, lda, Wl, n1, 8 * ti, 8 * tj, nq4, n1, n, lane);
      tj += nwarp;
    }
  }
  __syncthreads();
  if (warp == 0) { if (chol_diag8(A, lda, invd, Ms, kCsNB, 0, min(kCsNB, n), lane)) fail = 1; }
  __syncthreads();
  for (int k0 = 0; k0 < n; k0 += kCsNB) {
    const int nb = min(kCsNB, n - k0), nxt = k0 + nb;
    // rows below the (already factored) diagonal block -- rest of the leaf block + every extra row: a L_d^T = x, one row per thread
    for (int r = nxt + tid; r < n1; r += nt) {
      double a[kCsNB];
      double *ar = A + (size_t)r * lda + k0;
#pragma unroll
      for (int c = 0; c < kCsNB; c++) a[c] = (c < nb) ? ar[c] * invd[k0 + c] : 0.0;
#pragma unroll
      for (int c = 1; c < kCsNB; c++) {
        double s_ = a[c];
#pragma unroll
        for (int k = 0; k < c; k++) s_ = fma(-a[k], Ms[c * kCsNB + k], s_);
        a[c] = s_;
      }
#pragma unroll
      for (int c = 0; c < kCsNB; c++) { if (c < nb) ar[c] = a[c]; P[c * ldp + (r - k0)] = a[c]; }
    }
    __syncthreads();
    if (nxt >= n) break;
    const int pmax = n1 - 1 - k0, nb2 = min(kCsNB, n - nxt);
    const int Tr = (n1 - nxt + 7) >> 3, Tc = (n - nxt + 7) >> 3;
    // look-ahead: the tile column of the next panel first (all warps) ...
    for (int ti = warp; ti < Tr; ti += nwarp) leaf_tile8(A, lda, P, ldp, nxt + 8 * ti, nxt, nb + 8 * ti, nb, pmax, n1, n, lane);
    __syncthreads();
    // ... then warp 0 factors the next diagonal block (a pure latency chain) while the other warps update the rest
    if (warp == 0) { if (chol_diag8(A, lda, invd, Ms, kCsNB, nxt, nb2, lane)) fail = 1; }
    else {
      for (int ti = 1, tj = warp - 1;; ) {   // row tile ti >= 1 has column tiles 1 .. min(ti, Tc - 1)
        while (ti < Tr && tj >= min(ti, Tc - 1)) { tj -= min(ti, Tc - 1); ti++; }
        if (ti >= Tr) break;
        leaf_tile8(A, lda, P, ldp, nxt + 8 * ti, nxt + 8 * (tj + 1), nb + 8 * ti, nb + 8 * (tj + 1), pmax, n1, n, lane);
        tj += nwarp - 1;
      }
    }
    __syncthreads();
  }
  if (fail) { if (tid == 0) ctl->chol_fail = 1; return; }
  // L and 1/diag(L) for the back substitution; Y (transposed extra rows) into its rows of Wt, hub columns + rhs column
  double *Lg = d.leafL + lf.offL;
  for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; Lg[e] = j <= i ? A[(size_t)i * lda + j] : 0.0; }
  for (int e = tid; e < n; e += nt) Lg[(size_t)n * n + e] = invd[e];
  double *Yg = d.Wt + w.offW + (size_t)lf.row0 * w.ldw + w.hub0;
  for (int e = tid; e < n * (nh + 1); e += nt) {
    const int k = e / (nh + 1), c = e - k * (nh + 1);
    Yg[(size_t)k * w.ldw + c] = A[(size_t)(n + c) * lda + k];
  }
}

// Leaf part of the Gauss-Newton step: L^T x_b = z_b - Y_b x_hub, one CTA per (window, leaf)
constexpr int kLeafBackThreads = 128;
__host__ __device__ inline size_t leaf_back_smem_bytes(int n, int nh) { return ((size_t)n * n + 2 * (size_t)n + (size_t)nh + 8) * 8; }
__global__ void __launch_bounds__(kLeafBackThreads) k_leaf_back(Dev d) {
  const Leaf lf = d.leaf[blockIdx.x];
  const WinDesc &w = d.win[lf.win];
  Ctl *ctl = d.ctl + lf.win;
  if (ctl->done || ctl->reuse || ctl->chol_fail) return;
  extern __shared__ double sm[];
  const int n = lf.n, nh = w.n_hub;
  double *L = sm, *iv = L + (size_t)n * n, *v = iv + n, *xh = v + n;
  const double *Lg = d.leafL + lf.offL;
  const double *Yg = d.Wt + w.offW + (size_t)lf.row0 * w.ldw + w.hub0;
  double *gn = d.gn_c + w.offc;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int e = tid; e < n * n + n; e += nt) cp_async8(L + e, Lg + e);   // iv follows L in both layouts; lands during the products below
  for (int c = tid; c < nh; c += nt) xh[c] = -gn[w.hub0 + c];
  __syncthreads();
  for (int k0 = warp * 4; k0 < n; k0 += nwarp * 4) {   // four rows per pass: their loads are all in flight before the first reduction
    double s_[4] = {0.0, 0.0, 0.0, 0.0};
    const double *y0 = Yg + (size_t)k0 * w.ldw;
    for (int c0 = lane; c0 < nh; c0 += 96) {   // 4 rows x 3 column chunks: 12 independent loads before the first use
      double yv[3][4], xv[3];
#pragma unroll
      for (int u = 0; u < 3; u++) {
        const int c = c0 + 32 * u;
        xv[u] = c < nh ? xh[c] : 0.0;
#pragma unroll
        for (int q = 0; q < 4; q++) yv[u][q] = (c < nh && k0 + q < n) ? y0[(size_t)q * w.ldw + c] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 3; u++)
#pragma unroll
        for (int q = 0; q < 4; q++) s_[q] = fma(yv[u][q], xv[u], s_[q]);
    }
    const double zq = (lane < 4 && k0 + lane < n) ? y0[(size_t)lane * w.ldw + nh] : 0.0;   // z entries of the four rows
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const double t = warp_sum(s_[q]);
      const double z = __shfl_sync(0xffffffffu, zq, q);
      if (lane == 0 && k0 + q < n) v[k0 + q] = z - t;
    }
  }
  cp_async_wait_all();
  __syncthreads();
  if (warp != 0) return;
  for (int i = n - 1; i >= 0; i--) {
    const double xi = v[i] * iv[i];
    for (int j = lane; j < i; j += 32) v[j] -= L[(size_t)i * n + j] * xi;
    if (lane == 0) gn[lf.col0 + i] = -xi;
    __syncwarp();
  }
}

__global__ void k_zero_leaf_rows(Dev d) {
  const WinDesc &w = d.win[blockIdx.x];
  if (!w.n_leaf) return;
  double *Yg = d.Wt + w.offW + (size_t)w.nl * w.ldw;
  const size_t tot = (size_t)(w.wt_rows - w.nl) * w.ldw;
  for (size_t e = threadIdx.x; e < tot; e += blockDim.x) Yg[e] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// Step kernel: one CTA per window.
constexpr int kStepThreads = 256;
template <bool LEAF>   // LEAF: windows with leaves (block-sparse landmark rows); the other instantiation handles the dense rows
__global__ void __launch_bounds__(kStepThreads, LEAF ? 4 : 3) k_step(Dev d, int max_nc) {
  const int wi = blockIdx.x;
  const WinDesc &w = d.win[wi];
  if ((w.n_leaf != 0) != LEAF) return;
  Ctl *ctl = d.ctl + wi;
  if (ctl->done) return;
  extern __shared__ double sm[];
  double *red = sm;               // 40
  double *uc = sm + 40;           // n_c : g / D^2
  double *dcs = uc + max_nc;      // n_c : GN camera step
  double *D2 = dcs + max_nc;      // n_c
  const int tid = threadIdx.x, nt = blockDim.x, warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const int cur = ctl->cur, cand = 1 - cur;
  const int n = w.n_c, nlc = w.n_lc, ld = w.ldh, nl = w.nl;
  const double *H = d.Hcc[cur] + w.offH;
  const double *gcv = d.gc[cur] + w.offc;
  const double *hl = d.hl + w.offlm, *glv = d.gl + w.offlm, *dinv = d.dinv + w.offlm;
  double *gn_c = d.gn_c + w.offc, *gn_l = d.gn_l + w.offlm;
  const SolverParams &P = d.prm;
  const double *D2g = d.D2c + w.offc, *ucg = d.uc + w.offc, *D2l = d.D2l + w.offlm, *wuv = d.wu + w.offlm;
  for (int i = tid; i < n; i += nt) { D2[i] = D2g[i]; uc[i] = ucg[i]; dcs[i] = gn_c[i]; }
  __syncthreads();
  if (!ctl->reuse) {
    // gradient tolerance (checked at the top of a trust-region iteration, on a fresh linearisation)
    double gm = fmax(ctl->gmax_c, __longlong_as_double((long long)ctl->gmax_l_bits));
    if (!P.fixed_mode && gm <= P.gtol) { if (tid == 0) { ctl->done = 1; ctl->term = 2; } return; }
    if (ctl->chol_fail) { if (tid == 0) ctl->step_valid = 0; return; }
    // landmark back-substitution and the landmark part of the Cauchy / dogleg dot products
    const double *Wt = d.Wt + w.offW;
    double s_gg = 0, s_uHu = 0, s_nn = 0, s_gdn = 0;
    for (int l0 = warp * 8; l0 < nl; l0 += nw * 8) {
      double a[8];
#pragma unroll
      for (int q = 0; q < 8; q++) a[q] = 0.0;
      if (!LEAF) {
        // dense rows (single-drone window): 4 rows x 3 column chunks = 12 independent loads in flight before the first use
        for (int c0 = lane; c0 < nlc; c0 += 96) {
          double dc[3];
#pragma unroll
          for (int u = 0; u < 3; u++) dc[u] = c0 + 32 * u < nlc ? dcs[c0 + 32 * u] : 0.0;
#pragma unroll
          for (int qh = 0; qh < 8; qh += 4) {
            const double *r0 = Wt + (size_t)(l0 + qh) * w.ldw;
            double v[3][4];
#pragma unroll
            for (int u = 0; u < 3; u++)
#pragma unroll
              for (int q = 0; q < 4; q++) v[u][q] = (c0 + 32 * u < nlc && l0 + qh + q < nl) ? r0[(size_t)q * w.ldw + c0 + 32 * u] : 0.0;
#pragma unroll
            for (int u = 0; u < 3; u++)
#pragma unroll
              for (int q = 0; q < 4; q++) a[qh + q] = fma(v[u][q], dc[u], a[qh + q]);
          }
        }
      } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
          if (l0 + q < nl) {
            const double *row = Wt + (size_t)(l0 + q) * w.ldw;
            for (unsigned long long m = d.lm_mask[w.offlm + l0 + q]; m; m &= m - 1) {   // only the column tiles the row has entries in
              const int c = (__ffsll((long long)m) - 1) * 32 + lane;
              if (c < nlc) a[q] += row[c] * dcs[c];
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 8; q++) a[q] = warp_sum(a[q]);
      if (lane < 8 && l0 + lane < nl) {
        const int l = l0 + lane;
        double aq = a[0];
#pragma unroll
        for (int q = 1; q < 8; q++) if (lane == q) aq = a[q];
        const double di = dinv[l], gt = Wt[(size_t)l * w.ldw + nlc];
        const double gnl = -di * (gt + aq);
        gn_l[l] = gnl;
        const double h = hl[l], g = glv[l], dl2 = D2l[l], ul = g / dl2;
        s_gg += g * ul;
        s_uHu += 2.0 * ul * wuv[l] + h * ul * ul;
        s_nn += gnl * gnl * dl2;
        s_gdn += g * gnl;
      }
    }
    for (int j = tid; j < n; j += nt) { s_nn += dcs[j] * dcs[j] * D2[j]; s_gdn += gcv[j] * dcs[j]; }
    s_gg = block_sum(s_gg, red); s_uHu = block_sum(s_uHu, red); s_nn = block_sum(s_nn, red); s_gdn = block_sum(s_gdn, red);
    if (tid == 0) {
      s_gg += ctl->gg_cam; s_uHu += ctl->uHu_cam;
      ctl->gg = s_gg; ctl->nn = s_nn; ctl->gdn = s_gdn; ctl->alpha = s_gg / s_uHu;
    }
    __syncthreads();
  }
  // ---- traditional dogleg
  const double gg = ctl->gg, nn = ctl->nn, gdn = ctl->gdn, alpha = ctl->alpha, radius = ctl->radius, mu = ctl->mu;
  const double gn_norm = sqrt(nn), g_norm = sqrt(gg);
  double c1, c2, step_norm;
  if (gn_norm <= radius) { c1 = 0; c2 = 1; step_norm = gn_norm; }
  else if (g_norm * alpha >= radius) { c1 = radius / g_norm; c2 = 0; step_norm = radius; }
  else {
    double b_dot_a = -alpha * gdn, a_sq = alpha * alpha * gg, bma = nn - 2 * b_dot_a + a_sq;
    double c = b_dot_a - a_sq, dd = sqrt(c * c + bma * (radius * radius - a_sq));
    double beta = (c <= 0) ? (dd - c) / bma : (radius * radius - a_sq) / (dd + c);
    c1 = alpha * (1 - beta); c2 = beta; step_norm = radius;
  }
  // model cost change from scalars: H gn = -g - mu D^2 gn (to solver precision)
  const double uHu = gg / alpha;
  const double sg = -c1 * gg + c2 * gdn;
  const double uHgn = -gg - mu * gdn, gnHgn = -gdn - mu * nn;
  const double sHs = c1 * c1 * uHu - 2.0 * c1 * c2 * uHgn + c2 * c2 * gnHgn;
  const double model_change = -(sg + 0.5 * sHs);
  if (!(model_change > 0.0) || !isfinite(model_change)) {
    if (tid == 0) { ctl->step_valid = 0; ctl->model_change = model_change; }
    return;
  }
  // ---- candidate state
  double *step_c = d.step_c + w.offc, *step_l = d.step_l + w.offlm;
  for (int i = tid; i < n; i += nt) { double s = -c1 * uc[i] + c2 * dcs[i]; step_c[i] = s; uc[i] = s; }
  __syncthreads();
  double xn = 0, dxn = 0;
  const double *x6 = d.x6[cur] + (size_t)w.off6 * 8;
  double *y6 = d.x6[cand] + (size_t)w.off6 * 8;
  double *R6 = d.R6[cand] + (size_t)w.off6 * 12;
  const int *col6 = d.col6 + w.off6;
  for (int b = tid; b < w.n6; b += nt) {
    const double *x = x6 + b * 8;
    double o[7];
    int c = col6[b];
    if (c >= 0) {
      pose_plus(x, uc + c, o);
      for (int q = 0; q < 7; q++) { double df = x[q] - o[q]; xn += x[q] * x[q]; dxn += df * df; }
    } else for (int q = 0; q < 7; q++) o[q] = x[q];
    for (int q = 0; q < 7; q++) y6[b * 8 + q] = o[q];
    q2R(qload(o + 3), R6 + b * 12);
  }
  const double *xsb = d.xsb[cur] + (size_t)w.offsb * 9;
  double *ysb = d.xsb[cand] + (size_t)w.offsb * 9;
  const int *colsb = d.colsb + w.offsb;
  for (int e = tid; e < w.nsb * 9; e += nt) {
    int c = colsb[e / 9];
    double x = xsb[e], s = c >= 0 ? uc[c + e % 9] : 0.0;
    ysb[e] = x + s;
    if (c >= 0) { xn += x * x; dxn += s * s; }
  }
  if (tid == 0 && w.has_td) {
    double x = d.xtd[cur][wi], s = w.td_col >= 0 ? uc[w.td_col] : 0.0;
    d.xtd[cand][wi] = x + s;
    if (w.td_col >= 0) { xn += x * x; dxn += s * s; }
  }
  const double *xlm = d.xlm[cur] + w.offlm;
  double *ylm = d.xlm[cand] + w.offlm;
  for (int l = tid; l < nl; l += nt) {
    double g = glv[l];
    double s = -c1 * g / D2l[l] + c2 * gn_l[l];
    step_l[l] = s;
    double x = xlm[l];
    ylm[l] = x + s;
    xn += x * x; dxn += s * s;
  }
  xn = block_sum(xn, red); dxn = block_sum(dxn, red);
  if (tid == 0) {
    ctl->x_norm2 = xn; ctl->dx_norm2 = dxn; ctl->model_change = model_change; ctl->step_norm = step_norm;
    ctl->step_valid = 1; ctl->cand_cost_proj = 0.0; ctl->cand_cost_misc = 0.0;
  }
}

// ------------------------------------------------------------------------------------------------
// Trust-region bookkeeping (TrustRegionMinimizer / DoglegStrategy, SURVEY appendix B): one small CTA per
// window.  Thread 0 takes the accept / reject decision; when the window then holds a fresh accepted
// linearisation all threads derive the vectors every later kernel of the next iteration needs:
// D_c^2 = clamp(diag Hcc), u_c = g_c / D_c^2, and the camera part of |g~|^2 and of the gradient max-norm.
constexpr int kCtlThreads = 128;
__device__ void control_decide(Ctl *c, const SolverParams &P, int init) {
  if (init) {
    c->cost = c->cand_cost_misc + c->cand_cost_proj;
    if (init == 1) c->initial_cost = c->cost;
    c->reuse = 0; c->chol_fail = 0; c->step_valid = 1; c->gmax_l_bits = 0ull;
    c->cand_cost_misc = 0; c->cand_cost_proj = 0;
    return;
  }
  if (c->done) return;
  if (!c->step_valid) {
    // linear solver failure or non-positive model decrease: StepIsInvalid -> mu *= 10
    if (!c->chol_fail && !c->reuse) c->mu = fmax(1e-8, 2.0 * c->mu / 10.0);  // the factorisation itself succeeded
    c->mu *= 10.0; c->reuse = 0; c->chol_fail = 0; c->iter++; c->lin_count++; c->invalid_run++;
    c->step_valid = 1; c->gmax_l_bits = 0ull;
    if (c->invalid_run >= 5 || c->mu > 10.0) { c->done = 1; c->term = 4; }
    else if (c->iter >= P.max_iter) { c->done = 1; c->term = 0; }
    return;
  }
  c->invalid_run = 0;
  if (!c->reuse) c->mu = fmax(1e-8, 2.0 * c->mu / 10.0);  // relax after a successful factorisation
  const double cand = c->cand_cost_misc + c->cand_cost_proj;
  c->iter++; c->lin_count++;
  if (!P.fixed_mode) {
    const double xn = sqrt(c->x_norm2), dxn = sqrt(c->dx_norm2);
    if (dxn <= P.ptol * (xn + P.ptol)) { c->done = 1; c->term = 3; c->iter--; c->lin_count--; return; }
    if (fabs(c->cost - cand) <= P.ftol * c->cost) { c->done = 1; c->term = 1; c->iter--; c->lin_count--; return; }
  }
  const double rel = (c->cost - cand) / c->model_change;
  if (rel > P.min_rel_decrease) {
    c->cur = 1 - c->cur; c->cost = cand; c->succ++;
    if (rel < 0.25) c->radius *= 0.5;
    if (rel > 0.75) c->radius = fmax(c->radius, 3.0 * c->step_norm);
    c->radius = fmin(P.max_radius, c->radius);
    c->reuse = 0; c->gmax_l_bits = 0ull;
  } else {
    c->radius *= 0.5; c->reuse = 1;
    if (c->radius < 1e-32) { c->done = 1; c->term = 4; }
  }
  if (!c->done && c->iter >= P.max_iter) { c->done = 1; c->term = 0; }
}

__global__ void __launch_bounds__(kCtlThreads) k_control(Dev d, int init) {
  const int wi = blockIdx.x;
  Ctl *c = d.ctl + wi;
  __shared__ double red[40];
  if (threadIdx.x == 0) control_decide(c, d.prm, init);
  __syncthreads();
  if (c->done || c->reuse) return;
  // fresh accepted linearisation in buffer `cur`
  const WinDesc &w = d.win[wi];
  const int n = w.n_c, ld = w.ldh, cur = c->cur;
  const double *H = d.Hcc[cur] + w.offH, *g = d.gc[cur] + w.offc;
  double *D2 = d.D2c + w.offc, *uc = d.uc + w.offc;
  double gg = 0, gm = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double dd = d2_of(H[(size_t)i * ld + i]), gi = g[i], u = gi / dd;
    D2[i] = dd; uc[i] = u; gg += gi * u; gm = fmax(gm, fabs(gi));
  }
  gg = block_sum(gg, red);
  gm = block_max(gm, red);
  if (threadIdx.x == 0) { c->gg_cam = gg; c->gmax_c = gm; c->uHu_cam = 0.0; }
}

// reset the per-sub-step trust-region state (a fresh ceres::Solve)
__global__ void k_tr_reset(Dev d, int first) {
  const int wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= d.n_win) return;
  Ctl *c = d.ctl + wi;
  c->radius = d.prm.initial_radius; c->mu = d.prm.mu0; c->reuse = 0; c->done = 0; c->term = 0; c->step_valid = 1;
  c->invalid_run = 0; c->iter = 0; c->chol_fail = 0; c->gmax_l_bits = 0ull;
  c->cand_cost_misc = 0; c->cand_cost_proj = 0;
  if (first) { c->cur = 0; c->succ = 0; c->lin_count = 0; }
}

// ------------------------------------------------------------------------------------------------
// ADMM consensus exchange (replaces broadcastData / waitForSync / updateGlobal,
// VINSConsenusSolver.cpp:11-120, ConsensusSolver.cpp:166-228): per slot sum of [p(3), vech(q q^T)(10), 1].
__global__ void k_cons_pack(Dev d, int n6_total, const int *blk_win) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n6_total) return;
  int s = d.slot6[b];
  if (s < 0) return;
  const int wi = blk_win[b];
  const double *x = d.x6[d.ctl[wi].cur] + (size_t)b * 8;
  double *o = d.cons_buf + (size_t)s * 14;
  atomicAdd(o + 0, x[0]); atomicAdd(o + 1, x[1]); atomicAdd(o + 2, x[2]);
  int k = 3;
  for (int i = 0; i < 4; i++)
    for (int j = i; j < 4; j++) atomicAdd(o + (k++), x[3 + i] * x[3 + j]);
  atomicAdd(o + 13, 1.0);
}

// principal eigenvector of a symmetric 4x4 (cyclic Jacobi), Utility::averageQuaterions (utils.hpp:213-228)
D2BA_DEV void eig4_principal(const double *Min, double *q) {
  double A[16], V[16];
  for (int i = 0; i < 16; i++) { A[i] = Min[i]; V[i] = (i % 5 == 0) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 30; sweep++) {
    double off = 0;
    for (int i = 0; i < 4; i++) for (int j = i + 1; j < 4; j++) off += A[i * 4 + j] * A[i * 4 + j];
    if (off < 1e-40) break;
    for (int p = 0; p < 4; p++)
      for (int r = p + 1; r < 4; r++) {
        double apq = A[p * 4 + r];
        if (apq == 0.0) continue;
        double tau = (A[r * 4 + r] - A[p * 4 + p]) / (2.0 * apq);
        double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
        double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
        for (int k = 0; k < 4; k++) { double a = A[k * 4 + p], b = A[k * 4 + r]; A[k * 4 + p] = c * a - s * b; A[k * 4 + r] = s * a + c * b; }
        for (int k = 0; k < 4; k++) { double a = A[p * 4 + k], b = A[r * 4 + k]; A[p * 4 + k] = c * a - s * b; A[r * 4 + k] = s * a + c * b; }
        for (int k = 0; k < 4; k++) { double a = V[k * 4 + p], b = V[k * 4 + r]; V[k * 4 + p] = c * a - s * b; V[k * 4 + r] = s * a + c * b; }
      }
  }
  int m = 0;
  for (int i = 1; i < 4; i++) if (A[i * 4 + i] > A[m * 4 + m]) m = i;
  for (int k = 0; k < 4; k++) q[k] = V[k * 4 + m];
}

__global__ void k_cons_apply(Dev d, int n6_total, const int *blk_win) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n6_total) return;
  int s = d.slot6[b];
  if (s < 0) return;
  const int wi = blk_win[b];
  const double *x = d.x6[d.ctl[wi].cur] + (size_t)b * 8;
  const double *o = d.cons_buf + (size_t)s * 14;
  double cnt = o[13];
  if (!(cnt > 0.5)) return;
  double *z = d.z6 + (size_t)b * 8;
  z[0] = o[0] / cnt; z[1] = o[1] / cnt; z[2] = o[2] / cnt;
  double M[16], q[4];
  int k = 3;
  for (int i = 0; i < 4; i++) for (int j = i; j < 4; j++) { M[i * 4 + j] = o[k]; M[j * 4 + i] = o[k]; k++; }
  if (cnt < 1.5) { q[0] = x[3]; q[1] = x[4]; q[2] = x[5]; q[3] = x[6]; }   // single holder: quats[0] returned as is
  else eig4_principal(M, q);
  // hemisphere of the local estimate (eigenvector sign is arbitrary)
  double dot = q[0] * x[3] + q[1] * x[4] + q[2] * x[5] + q[3] * x[6];
  double sg = dot < 0 ? -1.0 : 1.0;
  z[3] = sg * q[0]; z[4] = sg * q[1]; z[5] = sg * q[2]; z[6] = sg * q[3];
  // tilde += (1 + alpha) * Log(z^-1 x)   (ConsensusSolver.cpp:127-133; DeltaPose/tangentSpace of swarm_msgs)
  Q4 qz = qload(z + 3);
  double dd[3] = {x[0] - z[0], x[1] - z[1], x[2] - z[2]}, t[3], Rz[9];
  q2R(qz, Rz); mtv3(Rz, dd, t);
  // rotate with the inverse quaternion exactly like the oracle (q^-1 * v)
  Q4 qe = qmul(qinv(qz), qload(x + 3));
  double nv = sqrt(qe.x * qe.x + qe.y * qe.y + qe.z * qe.z), th[3] = {0, 0, 0};
  if (nv > 0) { double ang = 2.0 * atan2(nv, fabs(qe.w)), sgn = qe.w < 0 ? -1.0 : 1.0; th[0] = ang * sgn * qe.x / nv; th[1] = ang * sgn * qe.y / nv; th[2] = ang * sgn * qe.z / nv; }
  double *tl = d.tilde6 + (size_t)b * 6;
  const double f = 1.0 + d.prm.relaxation_alpha;
  for (int i = 0; i < 3; i++) { tl[i] += f * t[i]; tl[3 + i] += f * th[i]; }
}

// snapshot of the local-only parameters for the NormalPrior terms of this ADMM sub-step
__global__ void k_cons_refs(Dev d, int nsb9_total, int nl_total, const int *sb_win, const int *lm_win) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nsb9_total) { int wi = sb_win[i / 9]; d.sb_ref[i] = d.xsb[d.ctl[wi].cur][i]; }
  if (i < nl_total) { int wi = lm_win[i]; d.lm_ref[i] = d.xlm[d.ctl[wi].cur][i]; }
  if (i < d.n_win) d.td_ref[i] = d.xtd[d.ctl[i].cur][i];
}

// z := x, tilde := 0 at the start of a solve (ConsenusParamState::create, ConsensusSolver.hpp:31-44)
__global__ void k_cons_init(Dev d, int n6_total) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n6_total) return;
  for (int q = 0; q < 8; q++) d.z6[(size_t)b * 8 + q] = d.x6[0][(size_t)b * 8 + q];
  for (int q = 0; q < 6; q++) d.tilde6[(size_t)b * 6 + q] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// Build the 32-observation AoSoA tiles from the compact upload records (ObsJ + shared ObsAnchor): gathers the
// record of every tile slot (pair-major order), computes the unit-sphere tangent base of the factor
// constructor (projectionTwoFrameOneCamFactor.cpp:34-45) and writes [field][lane] planes.
__global__ void __launch_bounds__(128) k_build_tiles(const long long *raw_off, const int *tile_src, const int *tile_win, const double *xtd, double *obs, int n_tiles) {
  const int tile = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (tile >= n_tiles) return;
  const int src = tile_src[(size_t)tile * kTile + lane];
  double f[kObsFields];
#pragma unroll
  for (int k = 0; k < kObsFields; k++) f[k] = 0.0;
  if (src >= 0) {
    const int wi = tile_win[tile];
    const ObsJ &p = reinterpret_cast<const ObsJ *>((uintptr_t)raw_off[4 * wi])[src];   // per-window base pointers
    if (p.type != D2BA_PROJ_DEPTH_PRIOR) {
      const ObsAnchor &a0 = reinterpret_cast<const ObsAnchor *>((uintptr_t)raw_off[4 * wi + 1])[p.anchor];
      const ObsJm *pm = reinterpret_cast<const ObsJm *>((uintptr_t)raw_off[4 * wi + 2]);
      const ObsAnchorM *am = reinterpret_cast<const ObsAnchorM *>((uintptr_t)raw_off[4 * wi + 3]);
#pragma unroll
      for (int k = 0; k < 3; k++) { f[k] = a0.pts_i[k]; f[3 + k] = p.pts_j[k]; }
      if (pm) {
#pragma unroll
        for (int k = 0; k < 3; k++) { f[6 + k] = am[p.anchor].vel_i[k]; f[9 + k] = pm[src].vel_j[k]; }
        f[12] = am[p.anchor].td_i; f[13] = pm[src].td_j;
      } else { f[12] = xtd[wi]; f[13] = xtd[wi]; }   // motion not uploaded: every stamp equals the constant td (host-checked)
      const double n = sqrt(f[3] * f[3] + f[4] * f[4] + f[5] * f[5]);
      const double a[3] = {f[3] / n, f[4] / n, f[5] / n};
      double t[3] = {0, 0, 1};
      if (a[0] == 0.0 && a[1] == 0.0 && a[2] == 1.0) { t[0] = 1; t[2] = 0; }
      const double dt = a[0] * t[0] + a[1] * t[1] + a[2] * t[2];
      double b1[3] = {t[0] - a[0] * dt, t[1] - a[1] * dt, t[2] - a[2] * dt};
      const double n1 = sqrt(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2]);
      b1[0] /= n1; b1[1] /= n1; b1[2] /= n1;
      f[14] = b1[0]; f[15] = b1[1]; f[16] = b1[2];
      f[17] = a[1] * b1[2] - a[2] * b1[1]; f[18] = a[2] * b1[0] - a[0] * b1[2]; f[19] = a[0] * b1[1] - a[1] * b1[0];
      f[20] = (p.type == D2BA_PROJ_2F1C_DEPTH) ? 1.0 / p.depth : 0.0;
    } else {
      f[2] = 1.0; f[5] = 1.0; f[14] = 1.0; f[18] = 1.0;
      f[20] = 1.0 / p.depth;
    }
  } else {  // padding slot: harmless constants
    f[2] = 1.0; f[5] = 1.0; f[14] = 1.0; f[18] = 1.0; f[20] = 1.0;
  }
  double *ob = obs + (size_t)tile * kObsFields * kTile;
#pragma unroll
  for (int k = 0; k < kObsFields; k++) ob[k * kTile + lane] = f[k];
}
void launch_build_tiles(const long long *raw_off, const int *tile_src, const int *tile_win, const double *xtd, double *obs, int n_tiles, cudaStream_t s) {
  if (n_tiles > 0) k_build_tiles<<<(n_tiles + 3) / 4, 128, 0, s>>>(raw_off, tile_src, tile_win, xtd, obs, n_tiles);
}

// ------------------------------------------------------------------------------------------------
// Second stage of the marginalization: S (landmarks already eliminated) is split into kept / removed camera
// columns and the removed ones are eliminated with the exact inverse (Cholesky), Utility::schurComplement
// (d2common/include/d2common/utils.hpp:131-141):  A = S11 - S12 S22^-1 S21,  b = g1 - S12 S22^-1 g2.
__global__ void __launch_bounds__(256) k_marg_reduce(const double *S, int ld, int n, const int *keep_idx, int nk, const int *rem_idx, int nr,
                                                     double *A, double *b, int *fail_flag) {
  extern __shared__ double sm[];
  double *R = sm;                 // nr x nr (lower Cholesky of S22)
  double *X = sm + nr * nr;       // nr x (nk+1)
  const int tid = threadIdx.x, nt = blockDim.x, nk1 = nk + 1;
  auto Sat = [&](int i, int j) { return i >= j ? S[(size_t)i * ld + j] : S[(size_t)j * ld + i]; };
  for (int e = tid; e < nr * nr; e += nt) { int i = e / nr, j = e % nr; R[e] = Sat(rem_idx[i], rem_idx[j]); }
  for (int e = tid; e < nr * nk1; e += nt) { int i = e / nk1, j = e % nk1; X[e] = j < nk ? Sat(rem_idx[i], keep_idx[j]) : S[(size_t)n * ld + rem_idx[i]]; }
  __syncthreads();
  __shared__ int bad;
  if (tid == 0) bad = 0;
  for (int c = 0; c < nr; c++) {
    __syncthreads();
    const double dcc = R[c * nr + c];
    if (!(dcc > 0.0)) { if (tid == 0) bad = 1; }
    const double inv = 1.0 / sqrt(dcc > 0.0 ? dcc : 1.0);
    __syncthreads();
    for (int r = c + tid; r < nr; r += nt) R[r * nr + c] = (r == c) ? dcc * inv : R[r * nr + c] * inv;
    __syncthreads();
    for (int e = tid; e < (nr - c - 1) * (nr - c - 1); e += nt) {
      int r = c + 1 + e / (nr - c - 1), c2 = c + 1 + e % (nr - c - 1);
      if (c2 <= r) R[r * nr + c2] -= R[r * nr + c] * R[c2 * nr + c];
    }
  }
  __syncthreads();
  // X <- S22^-1 X, one right-hand-side column per thread
  for (int j = tid; j < nk1; j += nt) {
    for (int i = 0; i < nr; i++) { double s_ = X[i * nk1 + j]; for (int k = 0; k < i; k++) s_ -= R[i * nr + k] * X[k * nk1 + j]; X[i * nk1 + j] = s_ / R[i * nr + i]; }
    for (int i = nr - 1; i >= 0; i--) { double s_ = X[i * nk1 + j]; for (int k = i + 1; k < nr; k++) s_ -= R[k * nr + i] * X[k * nk1 + j]; X[i * nk1 + j] = s_ / R[i * nr + i]; }
  }
  __syncthreads();
  for (int e = tid; e < nk * nk1; e += nt) {
    int i = e / nk1, j = e % nk1;
    double s_ = j < nk ? Sat(keep_idx[i], keep_idx[j]) : S[(size_t)n * ld + keep_idx[i]];
    for (int k = 0; k < nr; k++) s_ -= Sat(keep_idx[i], rem_idx[k]) * X[k * nk1 + j];
    if (j < nk) A[(size_t)i * nk + j] = s_; else b[i] = s_;
  }
  if (tid == 0 && bad) *fail_flag = 1;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of the kernel on ONE device (context), while every handle asks
// for what ITS windows need: the cache is keyed by (device, kernel) and only ever raised, so a handle with small windows
// cannot pull the limit from under a live handle with large ones and a second device gets its own attribute.
template <typename K>
cudaError_t raise_smem_limit(K kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void *>, size_t> cur;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(mu);
  size_t &c = cur[std::make_pair(dev, (const void *)kernel)];
  if (bytes <= c) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) c = bytes;
  return e;
}

int launch_marg_reduce(const double *S, int ld, int n, const int *keep_idx, int nk, const int *rem_idx, int nr, double *A, double *b, int *fail_flag,
                       cudaStream_t s) {
  size_t smb = ((size_t)nr * nr + (size_t)nr * (nk + 1)) * 8;
  cudaError_t e = raise_smem_limit(k_marg_reduce, (size_t)(smb));
  if (e != cudaSuccess) return (int)e;
  k_marg_reduce<<<1, 256, smb, s>>>(S, ld, n, keep_idx, nk, rem_idx, nr, A, b, fail_flag);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// host-callable launchers (keeps <<<>>> syntax inside this translation unit)
void launch_state_prep(const Dev &d, int n6_total, int buf, cudaStream_t s) {
  if (n6_total > 0) k_state_prep<<<(n6_total + 127) / 128, 128, 0, s>>>(d, n6_total, buf);
}
// packed upload record (kImuPack) -> the full constant record imu_raw / k_imu_prep index (kImuStride); entries the factor
// never reads stay at the zero of the finalize-time memset
__global__ void k_imu_unpack(const double *pk, double *full, int n_imu) {
  const int f = blockIdx.x, t = threadIdx.x;
  if (f >= n_imu || t >= kImuPack) return;
  int dst;
  if (t < 17) dst = t;
  else if (t < 71) { const int q = t - 17; dst = 17 + (q / 6) * 15 + 9 + q % 6; }
  else {
    const int q = t - 71;
    int i = (int)((sqrt(8.0 * q + 1.0) - 1.0) * 0.5);
    while ((i + 1) * (i + 2) / 2 <= q) i++;
    while (i * (i + 1) / 2 > q) i--;
    dst = 17 + 225 + i * 15 + (q - i * (i + 1) / 2);
  }
  full[(size_t)f * kImuStride + dst] = pk[(size_t)f * kImuPack + t];
}
void launch_imu_prep(const Dev &d, const double *packed, double *full, int n_imu, cudaStream_t s) {
  if (n_imu > 0) k_imu_unpack<<<n_imu, 192, 0, s>>>(packed, full, n_imu);
  if (n_imu > 0) k_imu_prep<<<(n_imu + 31) / 32, 32, 0, s>>>(d, n_imu);
}
void launch_prior_prep(const Dev &d, cudaStream_t s) { k_prior_prep<<<d.n_win, 256, 0, s>>>(d); }

size_t misc_smem_bytes(int max_prior_m) { return (size_t)(40 + 3 * max_prior_m + 8) * 8; }
void launch_imu_raw(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s) {
  if (n_imu_total > 0) k_imu_raw<<<(n_imu_total + 31) / 32, 32, 0, s>>>(d, eval_cur, n_imu_total);
}
void launch_imu_acc(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s) {
  if (n_imu_total > 0) k_imu_lin<<<(n_imu_total + kImuWarps - 1) / kImuWarps, kImuWarps * 32, (size_t)kImuWarps * kImuWarpDoubles * 8, s>>>(d, eval_cur, n_imu_total);
}
void launch_imu_lin(const Dev &d, int eval_cur, int n_imu_total, cudaStream_t s) {
  launch_imu_raw(d, eval_cur, n_imu_total, s);
  launch_imu_acc(d, eval_cur, n_imu_total, s);
}
void launch_misc_lin(const Dev &d, int eval_cur, int max_prior_m, cudaStream_t s) {
  k_misc_lin<<<d.n_win, kMiscThreads, misc_smem_bytes(max_prior_m), s>>>(d, eval_cur);
}

template <int NCT, int KR>
static size_t proj_smem() { return (size_t)4 * (GC_SIZE + NCT * 8 * (kTile * KR + 4)) * 8; }

int configure_kernels(int max_rows, int max_nc, int max_prior_m) {
  cudaError_t e;
  e = raise_smem_limit(k_proj_lin<2, 2>, (size_t)(proj_smem<2, 2>())); if (e) return e;
  e = raise_smem_limit(k_proj_lin<4, 2>, (size_t)(proj_smem<4, 2>())); if (e) return e;
  e = raise_smem_limit(k_proj_lin<2, 4>, (size_t)(proj_smem<2, 4>())); if (e) return e;
  e = raise_smem_limit(k_proj_lin<4, 4>, (size_t)(proj_smem<4, 4>())); if (e) return e;
  e = raise_smem_limit(k_proj_lin_pp<true>, proj_pp_smem()); if (e) return e;
  e = raise_smem_limit(k_proj_lin_pp<false>, proj_pp_smem()); if (e) return e;
  // 4 x 51 KB per SM needs the large shared-memory carveout
  cudaFuncSetAttribute(k_proj_lin_pp<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_proj_lin_pp<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
#if D2BA_PP_BLOCKS > 4
  // 37 KB per CTA: the large shared-memory carveout lets the register file, not the L1 split, set the occupancy
  cudaFuncSetAttribute(k_proj_lin_pp<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_proj_lin_pp<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
#endif

  size_t chol = (size_t)(kNB * (max_rows + 4) + 2 * max_rows + 16 + 16 * 32 + kNB * (kNB + 1)) * 8;
  e = raise_smem_limit(k_chol, (size_t)(chol)); if (e) return e;
  size_t st = (size_t)(40 + 3 * max_nc) * 8;
  e = raise_smem_limit(k_step<false>, (size_t)(st)); if (e) return e;
  e = raise_smem_limit(k_step<true>, (size_t)(st)); if (e) return e;
  e = raise_smem_limit(k_misc_lin, (size_t)(misc_smem_bytes(max_prior_m))); if (e) return e;
  e = raise_smem_limit(k_imu_lin, (size_t)kImuWarps * kImuWarpDoubles * 8); if (e) return e;
  return 0;
}
// the row buffers of the per-landmark gather grow with the landmark-coupled width (multi-agent windows: 6 x 88 poses)
int configure_gather(int max_ldw) {
  cudaError_t e;
  e = raise_smem_limit(k_lm_gather, (size_t)kGatherWarps * max_ldw * 8); if (e) return e;
  e = raise_smem_limit(k_lm_gather16, (size_t)kG16Lm * max_ldw * 8); if (e) return e;
  return 0;
}

void launch_proj_lin(const Dev &d, int variant, int eval_cur, int job_begin, int job_count, cudaStream_t s) {
  if (job_count <= 0) return;
  int grid = (job_count + 3) / 4;
  switch (variant) {
    case 0: k_proj_lin<2, 2><<<grid, 128, proj_smem<2, 2>(), s>>>(d, eval_cur, job_begin, job_count); break;
    case 1: k_proj_lin<4, 2><<<grid, 128, proj_smem<4, 2>(), s>>>(d, eval_cur, job_begin, job_count); break;
    case 2: k_proj_lin<2, 4><<<grid, 128, proj_smem<2, 4>(), s>>>(d, eval_cur, job_begin, job_count); break;
    case 3: k_proj_lin<4, 4><<<grid, 128, proj_smem<4, 4>(), s>>>(d, eval_cur, job_begin, job_count); break;
    case 4: k_proj_lin_pp<true><<<grid, 128, proj_pp_smem(), s>>>(d, eval_cur, job_begin, job_count); break;
    case 5: k_proj_lin_pp<false><<<grid, 128, proj_pp_smem(), s>>>(d, eval_cur, job_begin, job_count); break;
  }
}
void launch_proj_debug(const Dev &d, double *out, int n_tiles, const int *tile_win, cudaStream_t s) {
  if (n_tiles > 0) k_proj_debug<<<n_tiles, 32, 0, s>>>(d, out, n_tiles, tile_win);
}
void launch_lm_gather(const Dev &d, const int *lm_win, int n_lm_total, int max_ldw, int any_compact, int any_wide, cudaStream_t s) {
  if (n_lm_total <= 0) return;
  if (any_wide)
    k_lm_gather<<<(n_lm_total + kGatherWarps - 1) / kGatherWarps, kGatherWarps * 32, (size_t)kGatherWarps * max_ldw * 8, s>>>(d, lm_win, n_lm_total, max_ldw);
  if (any_compact)
    k_lm_gather16<<<(n_lm_total + kG16Lm - 1) / kG16Lm, kG16Lm * 16, (size_t)kG16Lm * max_ldw * 8, s>>>(d, lm_win, n_lm_total, max_ldw);
}
void launch_schur_small(const Dev &d, int max_ldw, cudaStream_t s) {
  k_schur_small<<<d.n_win, kSsThreads, (size_t)(2 * 32 * (max_ldw + 4) + 40) * 8, s>>>(d);
}
int configure_schur_small(int max_ldw) {
  return (int)raise_smem_limit(k_schur_small, (size_t)((2 * 32 * (max_ldw + 4) + 40) * 8));
}
void launch_schur(const Dev &d, const void *tiles, int n_tiles, cudaStream_t s) {
  if (n_tiles > 0) k_schur<<<n_tiles, 128, 0, s>>>(d, reinterpret_cast<const SchurTile *>(tiles));
}
size_t leaf_elim_smem(int n, int n_hub) { return leaf_elim_smem_bytes(n, n_hub); }
size_t leaf_back_smem(int n, int n_hub) { return leaf_back_smem_bytes(n, n_hub); }
int leaf_max_cols() { return kLeafMaxCols; }
int configure_leaf_elim(size_t smem) { return (int)raise_smem_limit(k_leaf_elim, smem); }
int configure_leaf_back(size_t smem) { return (int)raise_smem_limit(k_leaf_back, smem); }
void launch_leaf_elim(const Dev &d, size_t smem, cudaStream_t s) { if (d.n_leaf_total > 0) k_leaf_elim<<<d.n_leaf_total, kLeafThreads, smem, s>>>(d); }
void launch_leaf_back(const Dev &d, size_t smem, cudaStream_t s) { if (d.n_leaf_total > 0) k_leaf_back<<<d.n_leaf_total, kLeafBackThreads, smem, s>>>(d); }
void launch_zero_leaf_rows(const Dev &d, cudaStream_t s) { k_zero_leaf_rows<<<d.n_win, 256, 0, s>>>(d); }
size_t chol_smem_need(int n) { return chol_smem_bytes(n); }
int configure_chol_smem(int max_n) {
  return (int)raise_smem_limit(k_chol_smem, (size_t)(chol_smem_bytes(max_n)));
}
void launch_chol_smem(const Dev &d, int max_n, cudaStream_t s) {
  // small systems (after the speed-bias elimination): 4 warps per window so that several windows share an SM
  const int threads = max_n <= 96 ? 128 : kCsThreads;
  k_chol_smem<<<d.n_win, threads, chol_smem_bytes(max_n), s>>>(d);
}
__global__ void k_zero_sb_rows(Dev d) {
  const WinDesc &w = d.win[blockIdx.x];
  if (!w.sb_elim) return;
  double *Yg = d.Wt + w.offW + (size_t)w.nl * w.ldw;
  const size_t tot = (size_t)(w.wt_rows - w.nl) * w.ldw;
  for (size_t e = threadIdx.x; e < tot; e += blockDim.x) Yg[e] = 0.0;
}
void launch_zero_sb_rows(const Dev &d, cudaStream_t s) { k_zero_sb_rows<<<d.n_win, 256, 0, s>>>(d); }
size_t sb_elim_smem(int ldw, int n_c, int nb) { return sbe_smem_bytes(ldw, n_c, nb); }
int configure_sb_elim(size_t smem) { return (int)raise_smem_limit(k_sb_elim, (size_t)(smem)); }
void launch_sb_elim(const Dev &d, size_t smem, cudaStream_t s) { k_sb_elim<<<d.n_win, kSeThreads, smem, s>>>(d); }
size_t sb_back_smem(int nlc, int nb) { return sb_back_smem_bytes(nlc, nb); }
int sb_max_blocks() { return kSeMaxBlocks; }
void launch_sb_back(const Dev &d, size_t smem, cudaStream_t s) { k_sb_back<<<d.n_win, kSbBackThreads, smem, s>>>(d); }
int configure_sb_back(size_t smem) { return (int)raise_smem_limit(k_sb_back, smem); }
void launch_chol(const Dev &d, int max_rows, cudaStream_t s) {
  size_t sm = (size_t)(kNB * (max_rows + 4) + 2 * max_rows + 16 + 16 * 32 + kNB * (kNB + 1)) * 8;
  k_chol<<<d.n_win, kCholThreads, sm, s>>>(d, max_rows);
}
void launch_step(const Dev &d, int max_nc, cudaStream_t s) {
  // both kinds of windows may share a handle: each instantiation skips the other's windows
  if (d.n_leaf_total < 0 || d.n_plain_win > 0) k_step<false><<<d.n_win, kStepThreads, (size_t)(40 + 3 * max_nc) * 8, s>>>(d, max_nc);
  if (d.n_leaf_total > 0) k_step<true><<<d.n_win, kStepThreads, (size_t)(40 + 3 * max_nc) * 8, s>>>(d, max_nc);
}
void launch_control(const Dev &d, int init, cudaStream_t s) { k_control<<<d.n_win, kCtlThreads, 0, s>>>(d, init); }
void launch_tr_reset(const Dev &d, int first, cudaStream_t s) { k_tr_reset<<<(d.n_win + 127) / 128, 128, 0, s>>>(d, first); }
void launch_cons_init(const Dev &d, int n6_total, cudaStream_t s) { if (n6_total > 0) k_cons_init<<<(n6_total + 127) / 128, 128, 0, s>>>(d, n6_total); }
void launch_cons_pack(const Dev &d, int n6_total, const int *blk_win, cudaStream_t s) { if (n6_total > 0) k_cons_pack<<<(n6_total + 127) / 128, 128, 0, s>>>(d, n6_total, blk_win); }
void launch_cons_apply(const Dev &d, int n6_total, const int *blk_win, cudaStream_t s) { if (n6_total > 0) k_cons_apply<<<(n6_total + 127) / 128, 128, 0, s>>>(d, n6_total, blk_win); }
void launch_cons_refs(const Dev &d, int nsb_total, int nl_total, const int *sb_win, const int *lm_win, cudaStream_t s) {
  int n = nsb_total * 9; if (nl_total > n) n = nl_total; if (d.n_win > n) n = d.n_win;
  if (n > 0) k_cons_refs<<<(n + 127) / 128, 128, 0, s>>>(d, nsb_total * 9, nl_total, sb_win, lm_win);
}

}  // namespace d2ba
