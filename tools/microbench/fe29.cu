// Experiment for round 2: GF(2^255-19) multiplication on 9 x 29-bit limbs with PLAIN 64-bit multiply-accumulates
// (IMAD.WIDE.U32 without the carry-in/out .X form, no carry chains during accumulation) versus the production
// 8 x 32-bit saturated-limb multiplier (fe_asm.cuh).  Same harness as febench.cu.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"
#include "../../hotstuff_b200/csrc/fe.cuh"
#define ITERS 2048
#define M29 0x1fffffffu
struct fe29 { uint32_t v[9]; };
__device__ __forceinline__ void fe29_mul(fe29 &r, const fe29 &a, const fe29 &b) {
  uint64_t c[17];
#pragma unroll
  for (int k = 0; k < 17; k++) c[k] = 0;
#pragma unroll
  for (int i = 0; i < 9; i++)
#pragma unroll
    for (int j = 0; j < 9; j++) c[i + j] += (uint64_t)a.v[i] * b.v[j];
  // carry-propagate the 17 columns to 29-bit limbs l[0..17]
  uint32_t l[18];
  uint64_t carry = 0;
#pragma unroll
  for (int k = 0; k < 17; k++) {
    uint64_t t = c[k] + carry;
    l[k] = (uint32_t)t & M29;
    carry = t >> 29;
  }
  l[17] = (uint32_t)carry;
  // fold: 2^261 = 1216 (mod p)
  carry = 0;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    uint64_t t = (uint64_t)l[k] + (uint64_t)l[k + 9] * 1216u + carry;
    r.v[k] = (uint32_t)t & M29;
    carry = t >> 29;
  }
  uint32_t t0 = r.v[0] + (uint32_t)carry * 1216u;  // carry < 2^12
  r.v[0] = t0 & M29;
  r.v[1] += t0 >> 29;
}
__device__ __forceinline__ void fe29_add(fe29 &r, const fe29 &a, const fe29 &b) {
#pragma unroll
  for (int k = 0; k < 9; k++) r.v[k] = a.v[k] + b.v[k];   // lazy: no carries
}
template <int KIND>
__global__ void __launch_bounds__(256) k(uint32_t *out, uint32_t seed) {
  uint32_t acc = 0;
  if (KIND == 0) {
    fe29 a, b, c;
    for (int i = 0; i < 9; i++) { a.v[i] = (seed * (i + 1) + threadIdx.x) & M29; b.v[i] = (seed * (i + 3) ^ threadIdx.x) & M29; c.v[i] = i; }
#pragma unroll 1
    for (int i = 0; i < ITERS; i++) { fe29_mul(c, a, b); fe29_mul(a, b, c); fe29_mul(b, c, a); fe29_mul(c, a, b); }
    for (int i = 0; i < 9; i++) acc ^= a.v[i] ^ b.v[i] ^ c.v[i];
  } else if (KIND == 1) {
    fe a, b, c;
    for (int i = 0; i < 8; i++) { a.v[i] = seed * (i + 1) + threadIdx.x; b.v[i] = seed * (i + 3) ^ threadIdx.x; c.v[i] = i + threadIdx.x; }
#pragma unroll 1
    for (int i = 0; i < ITERS; i++) { fe_mul(c, a, b); fe_mul(a, b, c); fe_mul(b, c, a); fe_mul(c, a, b); }
    for (int i = 0; i < 8; i++) acc ^= a.v[i] ^ b.v[i] ^ c.v[i];
  } else if (KIND == 2) {  // madd-like mix: 7 mul + 8 add per iteration, 29-bit (lazy adds)
    fe29 x, y, z, t;
    for (int i = 0; i < 9; i++) { x.v[i] = (seed * (i + 1) + threadIdx.x) & M29; y.v[i] = (seed * (i + 3) ^ threadIdx.x) & M29; z.v[i] = (i + 5 * threadIdx.x) & M29; t.v[i] = (seed + i) & M29; }
#pragma unroll 1
    for (int i = 0; i < ITERS / 2; i++) {
      fe29 a, b, c, d, e, f, g, h, u;
      fe29_add(u, y, x); fe29_mul(a, u, t); fe29_add(u, y, z); fe29_mul(b, u, x); fe29_mul(c, t, z); fe29_add(d, z, z);
      fe29_add(e, b, a); fe29_add(h, b, a); fe29_add(f, d, c); fe29_add(g, d, c);
      fe29_mul(x, e, f); fe29_mul(y, g, h); fe29_mul(z, f, g); fe29_mul(t, e, h);
    }
    for (int i = 0; i < 9; i++) acc ^= x.v[i] ^ y.v[i] ^ z.v[i] ^ t.v[i];
  } else {                 // same mix on the production representation
    fe x, y, z, t;
    for (int i = 0; i < 8; i++) { x.v[i] = seed * (i + 1) + threadIdx.x; y.v[i] = seed * (i + 3) ^ threadIdx.x; z.v[i] = i + 5 * threadIdx.x; t.v[i] = seed + i; }
#pragma unroll 1
    for (int i = 0; i < ITERS / 2; i++) {
      fe a, b, c, d, e, f, g, h, u;
      fe_sub(u, y, x); fe_mul(a, u, t); fe_add(u, y, z); fe_mul(b, u, x); fe_mul(c, t, z); fe_add(d, z, z);
      fe_sub(e, b, a); fe_add(h, b, a); fe_sub(f, d, c); fe_add(g, d, c);
      fe_mul(x, e, f); fe_mul(y, g, h); fe_mul(z, f, g); fe_mul(t, e, h);
    }
    for (int i = 0; i < 8; i++) acc ^= x.v[i] ^ y.v[i] ^ z.v[i] ^ t.v[i];
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
template <int KIND> void run(const char *name, int bps, double ops_per_iter) {
  uint32_t *out; int blocks = dev_sms() * bps, threads = 256;
  cudaMalloc(&out, blocks * threads * 4);
  k<KIND><<<blocks, threads>>>(out, 12345); cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0); k<KIND><<<blocks, threads>>>(out, 12345); cudaEventRecord(e1); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  printf("%-34s threads/SM=%4d  %.3f ms  %.3e field-muls/s\n", name, threads * bps, ms, ops_per_iter * threads * blocks / (ms * 1e-3));
  cudaFree(out);
}
int main() {
  for (int bps : {2, 4}) {
    run<0>("mul 9x29 plain IMAD.WIDE", bps, ITERS * 4.0);
    run<1>("mul 8x32 IMAD.WIDE.X (production)", bps, ITERS * 4.0);
    run<2>("madd mix 9x29 (7 mul + 8 lazy add)", bps, ITERS / 2 * 7.0);
    run<3>("madd mix 8x32 (production)", bps, ITERS / 2 * 7.0);
  }
}
