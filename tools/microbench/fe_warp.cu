// Warp-cooperative GF(2^255-19) multiplication with shuffle carry propagation — the layout BASELINE.json's north_star names ("warp-shuffle
// carry propagation for the 256-bit field arithmetic") — measured against the thread-per-element multiplier the engine ships (fe_asm.cuh).
// Eight lanes hold one field element (lane j = limb j); a warp multiplies four elements at a time:
//   products   lane j forms result columns j and j+8: a_i (broadcast shuffle) x b_((j-i) mod 8) (gather shuffle), 8 IMAD.WIDE per lane
//   fold       V_j = col_j + 38 col_(j+8)   (2^256 = 38 mod p), three 32-bit words per lane
//   carries    R_j = w0_j + w1_(j-1) + w2_(j-2) via shuffles (wrapping x38 at lane 0), then a shuffle ripple until no lane carries
// Reports throughput (all SMs busy) and lone-warp latency for both designs, after checking the cooperative product against fe_mul.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/microbench/fe_warp tools/microbench/fe_warp.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
#include "device.cuh"
#include "../../hotstuff_b200/csrc/fe.cuh"

__device__ __forceinline__ uint32_t coop_mul(uint32_t a, uint32_t b) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, gl = lane & 7, base = lane & 24;
  uint64_t Llo = 0, Hlo = 0, Lhi = 0, Hhi = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint32_t ai = __shfl_sync(full, a, base + i);
    const uint32_t bx = __shfl_sync(full, b, base + ((gl - i) & 7));
    const uint64_t p = (uint64_t)ai * bx;
    if (i <= gl) {
      Llo += (uint32_t)p;
      Hlo += p >> 32;
    } else {
      Lhi += (uint32_t)p;
      Hhi += p >> 32;
    }
  }
  uint64_t t0 = Llo + 38u * Lhi, t1 = Hlo + 38u * Hhi;
  const uint32_t w0 = (uint32_t)t0;
  t1 += t0 >> 32;
  const uint32_t w1 = (uint32_t)t1, w2 = (uint32_t)(t1 >> 32);
  uint64_t up1 = __shfl_sync(full, w1, base + ((gl + 7) & 7));
  uint64_t up2 = __shfl_sync(full, w2, base + ((gl + 6) & 7));
  if (gl == 0) up1 *= 38u;
  if (gl <= 1) up2 *= 38u;
  uint64_t R = (uint64_t)w0 + up1 + up2;
  while (true) {
    uint64_t c = R >> 32;
    if (!__any_sync(full, c != 0)) break;
    R &= 0xffffffffu;
    uint64_t cin = __shfl_sync(full, (uint32_t)c, base + ((gl + 7) & 7));  // c < 2^32 always (R < 2^41)
    if (gl == 0) cin *= 38u;
    R += cin;
  }
  return (uint32_t)R;
}

template <int KIND>  // 0: cooperative, 1: thread per element
__global__ void __launch_bounds__(256) k_tput(uint32_t *out, int iters, uint32_t seed) {
  if (KIND == 0) {
    uint32_t a = seed * (threadIdx.x + 1) + blockIdx.x, b = seed ^ (threadIdx.x * 2654435761u);
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
      a = coop_mul(a, b);
      b = coop_mul(b, a);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a ^ b;
  } else {
    fe a, b;
    for (int i = 0; i < 8; i++) { a.v[i] = seed * (i + 1) + threadIdx.x; b.v[i] = seed * (i + 3) ^ threadIdx.x; }
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
      fe_mul(a, a, b);
      fe_mul(b, b, a);
    }
    uint32_t x = 0;
    for (int i = 0; i < 8; i++) x ^= a.v[i] ^ b.v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = x;
  }
}
__global__ void k_lat(uint32_t *out, unsigned long long *cyc, uint32_t seed) {
  uint32_t a = seed * (threadIdx.x + 1), b = seed ^ (threadIdx.x * 2654435761u);
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++) a = coop_mul(a, b);
  unsigned long long t1 = clock64();
  out[threadIdx.x] = a;
  if (threadIdx.x == 0) cyc[0] = (t1 - t0) / 256;
}
// correctness: the cooperative product equals fe_mul modulo p on random and all-ones inputs
__global__ void k_check(uint32_t *bad, uint32_t seed) {
  const int lane = threadIdx.x & 31, gl = lane & 7, base = lane & 24;
  uint32_t x = seed * (threadIdx.x + 17) * 2654435761u, y = (seed + threadIdx.x) * 40503u ^ 0x9e3779b9u;
  if (blockIdx.x == 0) x = y = 0xffffffffu;
  if (blockIdx.x == 1) { x = 0xffffffffu; y = (gl == 7) ? 0x7fffffffu : 0xffffffedu; }
  const uint32_t r = coop_mul(x, y);
  fe A, B, C, D;
  for (int i = 0; i < 8; i++) {
    A.v[i] = __shfl_sync(0xffffffffu, x, base + i);
    B.v[i] = __shfl_sync(0xffffffffu, y, base + i);
    D.v[i] = __shfl_sync(0xffffffffu, r, base + i);
  }
  fe_mul(C, A, B);
  if (!fe_eq(C, D)) atomicAdd(bad, 1u);
}
int main() {
  uint32_t *out, *bad; unsigned long long *cyc;
  cudaMalloc(&out, (size_t)dev_sms() * 8 * 256 * 4); cudaMalloc(&bad, 4); cudaMalloc(&cyc, 8); cudaMemset(bad, 0, 4);
  k_check<<<64, 256>>>(bad, 12345u); k_check<<<64, 256>>>(bad, 777u);
  uint32_t hbad = 1; cudaMemcpy(&hbad, bad, 4, cudaMemcpyDeviceToHost);
  printf("cooperative product vs fe_mul: %u mismatching groups of %d\n", hbad, 2 * 64 * 256);
  const int iters = 2000;
  for (int kind = 0; kind < 2; kind++)
    for (int bps : {2, 4, 8}) {
      const int blocks = dev_sms() * bps;
      cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
      if (kind == 0) k_tput<0><<<blocks, 256>>>(out, 10, 5); else k_tput<1><<<blocks, 256>>>(out, 10, 5);
      cudaDeviceSynchronize();
      cudaEventRecord(e0);
      if (kind == 0) k_tput<0><<<blocks, 256>>>(out, iters, 5); else k_tput<1><<<blocks, 256>>>(out, iters, 5);
      cudaEventRecord(e1); cudaDeviceSynchronize();
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      const double muls = (double)iters * 2 * blocks * 256 / (kind == 0 ? 8 : 1);
      printf("%-38s threads/SM=%4d  %.3e field multiplications/s\n", kind == 0 ? "warp-cooperative (8 lanes, shuffles)" : "thread per element (fe_asm.cuh)", bps * 256, muls / (ms * 1e-3));
    }
  k_lat<<<1, 32>>>(out, cyc, 99); cudaDeviceSynchronize();
  unsigned long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
  printf("lone warp, dependent cooperative multiplications: %llu cycles each (thread-per-element fe_mul: ~520, tools/microbench/latency.cu)\n", h);
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
  return hbad != 0;
}
