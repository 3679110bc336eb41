// Throughput of the field primitives (mul / sqr / add / sub) in lane-ops per clk per SM.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"
#include "../../hotstuff_b200/csrc/fe.cuh"
#define ITERS 2048
template <int KIND>
__global__ void __launch_bounds__(256) k(uint32_t *out, unsigned long long *cyc, uint32_t seed) {
  fe a, b, c;
  for (int i = 0; i < 8; i++) { a.v[i] = seed * (i + 1) + threadIdx.x; b.v[i] = seed * (i + 3) ^ threadIdx.x; c.v[i] = i; }
  __syncthreads();
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < ITERS; i++) {
    if (KIND == 0) { fe_mul(c, a, b); fe_mul(a, b, c); fe_mul(b, c, a); fe_mul(c, a, b); }
    if (KIND == 1) { fe_sqr(a, a); fe_sqr(b, b); fe_sqr(c, c); fe_sqr(a, a); }
    if (KIND == 2) { fe_add(c, a, b); fe_add(a, b, c); fe_add(b, c, a); fe_add(c, a, b); }
    if (KIND == 3) { fe_sub(c, a, b); fe_sub(a, b, c); fe_sub(b, c, a); fe_sub(c, a, b); }
  }
  unsigned long long t1 = clock64();
  uint32_t acc = 0;
  for (int i = 0; i < 8; i++) acc ^= a.v[i] ^ b.v[i] ^ c.v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int KIND> void run(const char *name, int threads, int bps) {
  uint32_t *out; unsigned long long *cyc; int blocks = dev_sms() * bps;
  cudaMalloc(&out, blocks * threads * 4); cudaMalloc(&cyc, blocks * 8);
  k<KIND><<<blocks, threads>>>(out, cyc, 12345); cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0); k<KIND><<<blocks, threads>>>(out, cyc, 12345); cudaEventRecord(e1); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double ops = (double)ITERS * 4.0 * threads * blocks;
  printf("%-8s threads/SM=%4d  %.3f ms  %.3e ops/s  (%.1f clk/SM per lane-op at the maximum SM clock)\n", name, threads * bps, ms, ops / (ms * 1e-3),
         dev_clock_hz() * blocks / bps / (ops / (ms * 1e-3)));
  cudaFree(out); cudaFree(cyc);
}
int main() {
  for (int bps : {1, 2, 4, 8}) { run<0>("fe_mul", 256, bps); run<1>("fe_sqr", 256, bps); run<2>("fe_add", 256, bps); run<3>("fe_sub", 256, bps); }
}
