// d2ba_math.cuh -- small fixed-size fp64 helpers for the device code.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace d2ba {

#define D2BA_DEV __device__ __forceinline__

struct Q4 { double x, y, z, w; };

D2BA_DEV Q4 qmul(const Q4 &a, const Q4 &b) {
  Q4 r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
  r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
  return r;
}
D2BA_DEV Q4 qinv(const Q4 &a) {  // conjugate / |a|^2 (Eigen inverse())
  double n2 = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
  double s = 1.0 / n2;
  return Q4{-a.x * s, -a.y * s, -a.z * s, a.w * s};
}
D2BA_DEV Q4 qpos(const Q4 &q) { return q.w >= 0.0 ? q : Q4{-q.x, -q.y, -q.z, -q.w}; }
D2BA_DEV Q4 qload(const double *p) { return Q4{p[0], p[1], p[2], p[3]}; }

// rotation matrix of a quaternion, row-major (same polynomial as Eigen::toRotationMatrix)
D2BA_DEV void q2R(const Q4 &q, double *R) {
  double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

D2BA_DEV void mv3(const double *A, const double *v, double *o) {  // o = A v
  double a = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
  double b = A[3] * v[0] + A[4] * v[1] + A[5] * v[2];
  double c = A[6] * v[0] + A[7] * v[1] + A[8] * v[2];
  o[0] = a; o[1] = b; o[2] = c;
}
D2BA_DEV void mtv3(const double *A, const double *v, double *o) {  // o = A^T v
  double a = A[0] * v[0] + A[3] * v[1] + A[6] * v[2];
  double b = A[1] * v[0] + A[4] * v[1] + A[7] * v[2];
  double c = A[2] * v[0] + A[5] * v[1] + A[8] * v[2];
  o[0] = a; o[1] = b; o[2] = c;
}
D2BA_DEV void mm3(const double *A, const double *B, double *C) {  // C = A B
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
D2BA_DEV void mtm3(const double *A, const double *B, double *C) {  // C = A^T B
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C[i * 3 + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
D2BA_DEV void mmt3(const double *A, const double *B, double *C) {  // C = A B^T
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C[i * 3 + j] = A[i * 3] * B[j * 3] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}
D2BA_DEV void cross3(const double *a, const double *b, double *o) {
  double t0 = a[1] * b[2] - a[2] * b[1], t1 = a[2] * b[0] - a[0] * b[2], t2 = a[0] * b[1] - a[1] * b[0];
  o[0] = t0; o[1] = t1; o[2] = t2;
}
D2BA_DEV double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// row (1x3) times 3x3: o = r^T M
D2BA_DEV void rm3(const double *r, const double *M, double *o) {
  double a = r[0] * M[0] + r[1] * M[3] + r[2] * M[6];
  double b = r[0] * M[1] + r[1] * M[4] + r[2] * M[7];
  double c = r[0] * M[2] + r[1] * M[5] + r[2] * M[8];
  o[0] = a; o[1] = b; o[2] = c;
}

// trust-region metric: D^2 = clamp(sqrt(h), 1e-6, 1e32)^2   (dogleg_strategy diagonal_)
D2BA_DEV double d2_of(double h) {
  double d = sqrt(h);
  d = d < 1e-6 ? 1e-6 : (d > 1e32 ? 1e32 : d);
  return d * d;
}

// 1/sqrt(d) to full double precision: fp32 MUFU seed + two Newton steps (22 -> 44 -> 88 bits); d must be a normal
// positive number in the float range (true for the pivots of the scaled normal equations)
D2BA_DEV double fast_rsqrt(double d) {
  double y = (double)rsqrtf((float)d);
  const double hd = 0.5 * d;
  y = y * (1.5 - hd * y * y);
  y = y * (1.5 - hd * y * y);
  return y;
}

D2BA_DEV double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum, result valid in every thread; `red` has >= 33 doubles of shared memory
D2BA_DEV double block_sum(double v, double *red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    double t = lane < nw ? red[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}
D2BA_DEV double block_max(double v, double *red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    double t = lane < nw ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmax(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// fp64 tensor-core MMA: D(8x8) += A(8x4) * B(4x8).  Fragment ownership: a = A[lane/4][lane%4],
// b = B[lane%4][lane/4], c0/c1 = C[lane/4][2*(lane%4) + {0,1}].
D2BA_DEV void dmma(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier helpers for shared-memory staging pipelines
D2BA_DEV unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
D2BA_DEV void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
D2BA_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
D2BA_DEV void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
D2BA_DEV void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 8-byte asynchronous global -> shared copy (LDGSTS): no register round trip, any number in flight
D2BA_DEV void cp_async8(void *dst_smem, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
D2BA_DEV void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
D2BA_DEV void mbar_arrive(unsigned long long *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
D2BA_DEV void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
D2BA_DEV unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
D2BA_DEV void mbar_wait(unsigned long long *bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  } while (!ok);
}

// PoseLocalParameterization::Plus: p += dp; q = normalize(q * [1, dtheta/2])
D2BA_DEV void pose_plus(const double *x, const double *d, double *o) {
  o[0] = x[0] + d[0]; o[1] = x[1] + d[1]; o[2] = x[2] + d[2];
  Q4 q = qmul(qload(x + 3), Q4{0.5 * d[3], 0.5 * d[4], 0.5 * d[5], 1.0});
  double n = 1.0 / sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  o[3] = q.x * n; o[4] = q.y * n; o[5] = q.z * n; o[6] = q.w * n;
}

}  // namespace d2ba
