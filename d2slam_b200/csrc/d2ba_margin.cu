// d2ba_margin.cu -- prior construction on the device.
//
//   toJacRes  (d2vins/src/factors/prior_factor.cpp:132-177): A <- (A + A^T)/2, A = V diag(s) V^T,
//             s <= 1e-8 -> 0, J = sqrt(S) V^T, e0 = sqrt(S^-1) V^T b.
// The symmetric eigen-decomposition is a one-CTA parallel-ordered (round-robin) two-sided Jacobi in
// fp64: each step applies m/2 disjoint rotations, columns first and then rows.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/d2ba.h"
#include "d2ba_launch.cuh"

namespace d2ba {

constexpr int kEigThreads = 1024;

}  // namespace d2ba

namespace d2ba {
// Batched toJacRes: one CTA per window whose prior was given in information form.  In place:
// Aio (m x m) holds A on entry and J on exit; bio (m) holds b on entry and e0 on exit; V is scratch (m x m).
__global__ void __launch_bounds__(kEigThreads) k_prior_from_info(const int *m_of, const long long *offJ, const long long *offv,
                                                                const int *is_info, double *Aall, double *Vall, double *ball) {
  const int wi = blockIdx.x;
  const int m = m_of[wi];
  if (m <= 0 || !is_info[wi]) return;
  double *A = Aall + offJ[wi], *V = Vall + offJ[wi], *b = ball + offv[wi];
  const int tid = threadIdx.x, nt = blockDim.x;
  extern __shared__ double smx[];
  double *cs = smx;                                  // 2 * half
  int *pq = reinterpret_cast<int *>(smx + m + 2);    // 2 * half ints
  double *ev = smx + 2 * (m + 2);                    // m eigenvalues
  double *bb = ev + m;                               // m
  __shared__ double s_off, s_diag;
  const int mp = (m + 1) / 2 * 2, half = mp / 2;
  // symmetrise, V = I
  for (int e = tid; e < m * m; e += nt) { int i = e / m, j = e % m; if (j < i) { double v = 0.5 * (A[i * m + j] + A[j * m + i]); A[i * m + j] = v; A[j * m + i] = v; } V[e] = (i == j) ? 1.0 : 0.0; }
  for (int i = tid; i < m; i += nt) bb[i] = b[i];
  __syncthreads();
  for (int sweep = 0; sweep < 60; sweep++) {
    if (tid == 0) { s_off = 0; s_diag = 0; }
    __syncthreads();
    double off = 0, dg = 0;
    for (int e = tid; e < m * m; e += nt) { int i = e / m, j = e % m; double v = A[e]; if (i == j) dg += v * v; else off += v * v; }
    for (int o = 16; o > 0; o >>= 1) { off += __shfl_xor_sync(0xffffffffu, off, o); dg += __shfl_xor_sync(0xffffffffu, dg, o); }
    if ((tid & 31) == 0) { atomicAdd(&s_off, off); atomicAdd(&s_diag, dg); }
    __syncthreads();
    if (s_off <= 1e-30 * (s_diag + s_off) || s_off == 0.0) break;
    for (int step = 0; step < mp - 1; step++) {
      for (int k = tid; k < half; k += nt) {
        int a = (k == 0) ? mp - 1 : (step + k) % (mp - 1);
        int bq = (step + mp - 1 - k) % (mp - 1);
        int p = a < bq ? a : bq, q = a < bq ? bq : a;
        double c = 1.0, s = 0.0;
        if (q < m) {
          double apq = A[p * m + q];
          if (apq != 0.0) {
            double tau = (A[q * m + q] - A[p * m + p]) / (2.0 * apq);
            double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
            c = 1.0 / sqrt(1.0 + t * t); s = t * c;
          }
        } else { q = -1; }
        cs[2 * k] = c; cs[2 * k + 1] = s; pq[2 * k] = p; pq[2 * k + 1] = q;
      }
      __syncthreads();
      for (int e = tid; e < half * m; e += nt) {
        int k = e / m, r = e % m;
        int p = pq[2 * k], q = pq[2 * k + 1];
        if (q < 0) continue;
        double c = cs[2 * k], s = cs[2 * k + 1];
        double ap = A[r * m + p], aq = A[r * m + q];
        A[r * m + p] = c * ap - s * aq; A[r * m + q] = s * ap + c * aq;
        double vp = V[r * m + p], vq = V[r * m + q];
        V[r * m + p] = c * vp - s * vq; V[r * m + q] = s * vp + c * vq;
      }
      __syncthreads();
      for (int e = tid; e < half * m; e += nt) {
        int k = e / m, r = e % m;
        int p = pq[2 * k], q = pq[2 * k + 1];
        if (q < 0) continue;
        double c = cs[2 * k], s = cs[2 * k + 1];
        double ap = A[p * m + r], aq = A[q * m + r];
        A[p * m + r] = c * ap - s * aq; A[q * m + r] = s * ap + c * aq;
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < m; i += nt) ev[i] = A[i * m + i];
  __syncthreads();
  // J[i][k] = sqrt(s_i) V[k][i];  e0[i] = sqrt(1/s_i) sum_k V[k][i] b[k]   (prior_factor.cpp:139-150)
  const double eps = 1e-8;
  for (int e = tid; e < m * m; e += nt) { int i = e / m, k = e % m; double s = ev[i] > eps ? sqrt(ev[i]) : 0.0; A[e] = s * V[k * m + i]; }
  for (int i = tid; i < m; i += nt) {
    double dot = 0;
    for (int k = 0; k < m; k++) dot += V[k * m + i] * bb[k];
    b[i] = (ev[i] > eps ? sqrt(1.0 / ev[i]) : 0.0) * dot;
  }
}

void launch_prior_from_info(const LaunchSummary &L, const int *m_of, const long long *offJ, const long long *offv, const int *is_info,
                            double *A, double *V, double *b, cudaStream_t s) {
  if (!L.any_info) return;
  size_t sm = (size_t)(4 * (L.max_prior_m + 2) + 8) * 8;
  k_prior_from_info<<<L.n_used, kEigThreads, sm, s>>>(m_of, offJ, offv, is_info, A, V, b);
}
}  // namespace d2ba
