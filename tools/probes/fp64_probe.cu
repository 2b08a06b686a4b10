// Micro-benchmark of the fp64 building blocks the solver kernels are made of (run on the GPU box):
// DFMA throughput / latency, DMMA m8n8k4 throughput / latency, shuffle latency, MUFU-seeded rsqrt chain.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
template <int ILP> __global__ void k_dfma(double *out, int iters, long long *cyc) {
  double a[ILP]; const double x = 1.0000001, y = 1e-9;
  for (int i = 0; i < ILP; i++) a[i] = threadIdx.x + i;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int i = 0; i < ILP; i++) a[i] = fma(a[i], x, y);
  long long t1 = clock64();
  double s = 0; for (int i = 0; i < ILP; i++) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int ILP> __global__ void k_dmma(double *out, int iters, long long *cyc) {
  double c0[ILP], c1[ILP]; double a = 1.0 + threadIdx.x * 1e-9, b = 1e-9;
  for (int i = 0; i < ILP; i++) { c0[i] = i; c1[i] = -i; }
  long long t0 = clock64();
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int i = 0; i < ILP; i++) dmma(c0[i], c1[i], a, b);
  long long t1 = clock64();
  double s = 0; for (int i = 0; i < ILP; i++) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_shfl(double *out, int iters, long long *cyc) {
  double v = threadIdx.x;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) v = __shfl_sync(0xffffffffu, v, (threadIdx.x + 1) & 31);
  long long t1 = clock64();
  out[threadIdx.x] = v; if (threadIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_rsqrt(double *out, int iters, long long *cyc) {
  double d = 2.0 + threadIdx.x;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) { double y = (double)rsqrtf((float)d); const double hd = 0.5 * d; y = y * (1.5 - hd * y * y); y = y * (1.5 - hd * y * y); d = d + y; }
  long long t1 = clock64();
  out[threadIdx.x] = d; if (threadIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_lds(double *out, int iters, long long *cyc) {
  __shared__ double sm[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = (double)((i * 7 + 1) & 1023);
  __syncthreads();
  int idx = threadIdx.x;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) idx = (int)sm[idx] & 1023;
  long long t1 = clock64();
  out[threadIdx.x] = idx; if (threadIdx.x == 0) *cyc = t1 - t0;
}
template <typename F> void run(const char *name, F launch, double ops_per_thread_iter, int threads, int blocks, int iters) {
  double *out; long long *cyc, h = 0; cudaMalloc(&out, sizeof(double) * threads * blocks); cudaMalloc(&cyc, 8);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(out, iters, cyc, threads, blocks); cudaDeviceSynchronize();
  cudaEventRecord(e0); launch(out, iters, cyc, threads, blocks); cudaEventRecord(e1); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1); cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
  double total = ops_per_thread_iter * iters * (double)threads * blocks;
  printf("%-28s blocks %4d thr %4d: %8.3f ms  %8.2f Gop/s  cycles/iter(thread0) %.2f\n", name, blocks, threads, ms, total / ms * 1e-6, (double)h / iters);
  cudaFree(out); cudaFree(cyc);
}
int main() {
  const int it = 20000;
  run("dfma ILP1 1 warp", [](double *o, int i, long long *c, int t, int b) { k_dfma<1><<<b, t>>>(o, i, c); }, 1, 32, 1, it);
  run("dfma ILP8 1 warp", [](double *o, int i, long long *c, int t, int b) { k_dfma<8><<<b, t>>>(o, i, c); }, 8, 32, 1, it);
  run("dfma ILP8 16 warps/SM", [](double *o, int i, long long *c, int t, int b) { k_dfma<8><<<b, t>>>(o, i, c); }, 8, 512, 132, it);
  run("dfma ILP8 32 warps/SM", [](double *o, int i, long long *c, int t, int b) { k_dfma<8><<<b, t>>>(o, i, c); }, 8, 1024, 132, it);
  run("dmma ILP1 1 warp", [](double *o, int i, long long *c, int t, int b) { k_dmma<1><<<b, t>>>(o, i, c); }, 8, 32, 1, it);
  run("dmma ILP4 1 warp", [](double *o, int i, long long *c, int t, int b) { k_dmma<4><<<b, t>>>(o, i, c); }, 32, 32, 1, it);
  run("dmma ILP4 16 warps/SM", [](double *o, int i, long long *c, int t, int b) { k_dmma<4><<<b, t>>>(o, i, c); }, 32, 512, 132, it);
  run("dmma ILP4 32 warps/SM", [](double *o, int i, long long *c, int t, int b) { k_dmma<4><<<b, t>>>(o, i, c); }, 32, 1024, 132, it);
  run("shfl chain", [](double *o, int i, long long *c, int t, int b) { k_shfl<<<b, t>>>(o, i, c); }, 1, 32, 1, it);
  run("rsqrt(f32 seed + 2 newton)", [](double *o, int i, long long *c, int t, int b) { k_rsqrt<<<b, t>>>(o, i, c); }, 1, 32, 1, it);
  run("lds dependent chain", [](double *o, int i, long long *c, int t, int b) { k_lds<<<b, t>>>(o, i, c); }, 1, 32, 1, it);
  return 0;
}
