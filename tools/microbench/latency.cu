// Single-warp LATENCY of the building blocks of the latency path (k_verify_small / k_digest32_long): cycles for one warp alone on
// an SM.  Answers "where do the 70 us of a single verify go" and sizes the warp-cooperative alternatives.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/microbench/latency tools/microbench/latency.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"
#include "../../hotstuff_b200/csrc/verify_core.cuh"
#include "../experiments/fe10.cuh"   // ten-limb latency experiment (not part of the product)

__global__ void k_lat(uint32_t *out, unsigned long long *cyc, uint32_t seed) {
  fe a, b;
  for (int i = 0; i < 8; i++) { a.v[i] = seed * (i + 1) + threadIdx.x; b.v[i] = seed * (i + 3) ^ threadIdx.x; }
  unsigned long long t[12];
  t[0] = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++) fe_sqr(a, a);                  // dependent squarings (the sqrt / inversion chains)
  t[1] = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++) fe_mul(a, a, b);               // dependent multiplications
  t[2] = clock64();
  uint32_t enc[8];
  for (int i = 0; i < 8; i++) enc[i] = a.v[i];
  ge_ext P;
  uint32_t ok = ge_decompress(P, enc);                        // R decompression (warp 1 of k_verify_small)
  t[3] = clock64();
  uint32_t h[16], R[8], A[8], M[8];
  for (int i = 0; i < 8; i++) { R[i] = P.X.v[i]; A[i] = P.Y.v[i]; M[i] = a.v[i] ^ ok; }
  sha512_ram32(h, R, A, M);                                    // k-hash, one block
  t[4] = clock64();
  uint32_t k[8];
  sc_reduce512(k, h);
  t[5] = clock64();
  ge_ext acc, o;
  ge_identity(acc);
  ge_from_signed_niels(o, P.X, P.Y);
  for (int i = 0; i < 8; i++) o.X.v[i] ^= k[i];
#pragma unroll 1
  for (int s = 0; s < 5; s++) { ge_add_ext(acc, acc, o); o = acc; }   // the 5 levels of the lane tree (shuffles not included)
  t[6] = clock64();
  fe inv;
  fe_invert(inv, acc.Z);
  t[7] = clock64();
  fe10 q;
  fe10_from_fe(q, inv);
  t[8] = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++) fe10_sqr(q, q);
  t[9] = clock64();
  fe10 q2 = q;
#pragma unroll 1
  for (int i = 0; i < 256; i++) fe10_mul(q, q, q2);
  t[10] = clock64();
  for (int i = 0; i < 8; i++) enc[i] = q.v[i] ^ (q.v[i + 2] << 7);
  {  // the (p-5)/8 exponentiation of a decompression on ten limbs
    fe tt;
    for (int i = 0; i < 8; i++) tt.v[i] = enc[i];
    fe_pow_p58_lat(tt, tt);
    ok ^= tt.v[0];
  }
  t[11] = clock64();
  uint32_t x = ok;
  for (int i = 0; i < 8; i++) x ^= acc.X.v[i] ^ inv.v[i] ^ P.X.v[i];
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) for (int i = 0; i < 11; i++) cyc[i] = t[i + 1] - t[i];
}
__global__ void k_sha_chain(uint64_t *out, unsigned long long *cyc, const uint64_t *kwg) {
  __shared__ uint64_t kw[80 * 32];
  for (int i = threadIdx.x; i < 80 * 32; i += 32) kw[i] = kwg[i];
  __syncwarp();
  sha512_state s;
  sha512_init(s);
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int j = 0; j < 32; j++) sha512_compress_kw_strided(s, kw + j, 32);
  unsigned long long t1 = clock64();
  out[threadIdx.x] = s.h[0] ^ s.h[7];
  if (threadIdx.x == 0) cyc[0] = (t1 - t0) / 32;
}
int main() {
  uint32_t *out; unsigned long long *cyc; uint64_t *kw;
  cudaMalloc(&out, 4096); cudaMalloc(&cyc, 128); cudaMalloc(&kw, 80 * 32 * 8); cudaMemset(kw, 0x5a, 80 * 32 * 8);
  unsigned long long h[12];
  const char *names[11] = {"256 dependent fe_sqr", "256 dependent fe_mul", "ge_decompress", "sha512 one block", "sc_reduce512", "5 x ge_add_ext (tree levels)", "fe_invert",
                           "(convert)", "256 dependent fe10_sqr", "256 dependent fe10_mul", "pow (p-5)/8 on ten limbs"};
  for (int rep = 0; rep < 2; rep++) { k_lat<<<1, 32>>>(out, cyc, 77 + rep); cudaDeviceSynchronize(); }
  cudaMemcpy(h, cyc, 88, cudaMemcpyDeviceToHost);
  for (int i = 0; i < 11; i++) printf("%-32s %8llu cycles  (%.2f us at the maximum SM clock)%s\n", names[i], h[i], h[i] / (dev_clock_hz() * 1e-6), i < 2 ? "  [per op: /256]" : "");
  for (int rep = 0; rep < 2; rep++) { k_sha_chain<<<1, 32>>>((uint64_t *)out, cyc, kw); cudaDeviceSynchronize(); }
  cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost);
  printf("%-32s %8llu cycles per block (%.1f per round)\n", "sha512 rounds from K+W table", h[0], h[0] / 80.0);
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
}
