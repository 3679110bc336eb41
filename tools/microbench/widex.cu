// Is IMAD.WIDE.U32.X (carry-in/out) as fast as plain IMAD.WIDE.U32?  And what does IMAD.MOV cost next to it?
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"
#define ITERS 4096
template <int KIND>
__global__ void __launch_bounds__(512, 1) k(uint32_t *out, unsigned long long *cyc, uint32_t seed) {
  uint32_t x = seed + threadIdx.x, y = seed * 3 + threadIdx.x * 7 + 1;
  unsigned long long a0 = x, a1 = y, a2 = x + 1, a3 = y + 1, b0 = x + 2, b1 = y + 2, b2 = x + 3, b3 = y + 3;
  __syncthreads();
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < ITERS; i++) {
    if (KIND == 0) {  // two independent 4-long carry chains of wide mads
      asm volatile("{.reg .u32 l0,h0,l1,h1,l2,h2,l3,h3;\n\t"
                   "mov.b64 {l0,h0}, %0; mov.b64 {l1,h1}, %1; mov.b64 {l2,h2}, %2; mov.b64 {l3,h3}, %3;\n\t"
                   "mad.lo.cc.u32 l0, %4, %5, l0;\n\tmadc.hi.cc.u32 h0, %4, %5, h0;\n\t"
                   "madc.lo.cc.u32 l1, %4, %5, l1;\n\tmadc.hi.cc.u32 h1, %4, %5, h1;\n\t"
                   "madc.lo.cc.u32 l2, %4, %5, l2;\n\tmadc.hi.cc.u32 h2, %4, %5, h2;\n\t"
                   "madc.lo.cc.u32 l3, %4, %5, l3;\n\tmadc.hi.u32 h3, %4, %5, h3;\n\t"
                   "mov.b64 %0, {l0,h0}; mov.b64 %1, {l1,h1}; mov.b64 %2, {l2,h2}; mov.b64 %3, {l3,h3};}"
                   : "+l"(a0), "+l"(a1), "+l"(a2), "+l"(a3) : "r"(x), "r"(y));
      asm volatile("{.reg .u32 l0,h0,l1,h1,l2,h2,l3,h3;\n\t"
                   "mov.b64 {l0,h0}, %0; mov.b64 {l1,h1}, %1; mov.b64 {l2,h2}, %2; mov.b64 {l3,h3}, %3;\n\t"
                   "mad.lo.cc.u32 l0, %4, %5, l0;\n\tmadc.hi.cc.u32 h0, %4, %5, h0;\n\t"
                   "madc.lo.cc.u32 l1, %4, %5, l1;\n\tmadc.hi.cc.u32 h1, %4, %5, h1;\n\t"
                   "madc.lo.cc.u32 l2, %4, %5, l2;\n\tmadc.hi.cc.u32 h2, %4, %5, h2;\n\t"
                   "madc.lo.cc.u32 l3, %4, %5, l3;\n\tmadc.hi.u32 h3, %4, %5, h3;\n\t"
                   "mov.b64 %0, {l0,h0}; mov.b64 %1, {l1,h1}; mov.b64 %2, {l2,h2}; mov.b64 %3, {l3,h3};}"
                   : "+l"(b0), "+l"(b1), "+l"(b2), "+l"(b3) : "r"(y), "r"(x));
    } else if (KIND == 1) {  // 8 plain wide mads
#define OP(w, p, q) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(p), "r"(q));
      OP(a0, x, y) OP(a1, x, y) OP(a2, x, y) OP(a3, x, y) OP(b0, y, x) OP(b1, y, x) OP(b2, y, x) OP(b3, y, x)
#undef OP
    } else if (KIND == 2) {  // 8 plain wide mads + 8 IMAD.MOV-ish (mov through mad.lo with 1)
#define OP(w, p, q) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(p), "r"(q));
      OP(a0, x, y) OP(a1, x, y) OP(a2, x, y) OP(a3, x, y) OP(b0, y, x) OP(b1, y, x) OP(b2, y, x) OP(b3, y, x)
#undef OP
      asm volatile("mad.lo.u32 %0, %0, 1, %1;" : "+r"(x) : "r"(y));
      asm volatile("mad.lo.u32 %0, %0, 1, %1;" : "+r"(y) : "r"(x));
    } else if (KIND == 3) {  // 8 wide + 8 addc-chain ALU ops
#define OP(w, p, q) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(p), "r"(q));
      OP(a0, x, y) OP(a1, x, y) OP(a2, x, y) OP(a3, x, y) OP(b0, y, x) OP(b1, y, x) OP(b2, y, x) OP(b3, y, x)
#undef OP
      uint32_t p0 = x, p1 = y, p2 = x ^ 5, p3 = y ^ 9;
      asm volatile("add.cc.u32 %0, %0, %4;\n\taddc.cc.u32 %1, %1, %4;\n\taddc.cc.u32 %2, %2, %4;\n\taddc.u32 %3, %3, %4;" : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3) : "r"(y));
      asm volatile("add.cc.u32 %0, %0, %4;\n\taddc.cc.u32 %1, %1, %4;\n\taddc.cc.u32 %2, %2, %4;\n\taddc.u32 %3, %3, %4;" : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3) : "r"(x));
      x ^= p3; y ^= p2 ^ p1 ^ p0;
    }
  }
  unsigned long long t1 = clock64();
  unsigned long long acc = a0 ^ a1 ^ a2 ^ a3 ^ b0 ^ b1 ^ b2 ^ b3;
  out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)acc ^ (uint32_t)(acc >> 32) ^ x ^ y;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int KIND> void run(const char *name, int bps) {
  uint32_t *out; unsigned long long *cyc; int blocks = dev_sms() * bps, threads = 512;
  cudaMalloc(&out, blocks * threads * 4); cudaMalloc(&cyc, blocks * 8);
  k<KIND><<<blocks, threads>>>(out, cyc, 12345); cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0); k<KIND><<<blocks, threads>>>(out, cyc, 12345); cudaEventRecord(e1); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  unsigned long long h[1024]; cudaMemcpy(h, cyc, dev_sms() * sizeof(h[0]), cudaMemcpyDeviceToHost);
  double avg = 0; for (int i = 0; i < dev_sms(); i++) avg += (double)h[i]; avg /= dev_sms();
  printf("%-36s %.3f ms  wide-mads/clk/SM = %.2f\n", name, ms, (double)ITERS * 8.0 * threads * bps / (ms * 1e-3 * dev_clock_hz()) );
  cudaFree(out); cudaFree(cyc);
}
int main() { run<0>("IMAD.WIDE.U32.X chains", 1); run<1>("IMAD.WIDE.U32 plain", 1); run<2>("plain + 2 IMAD per 8", 1); run<3>("plain + 8 IADD3.X per 8", 1);
             run<0>("IMAD.WIDE.U32.X chains (1024 thr/SM)", 2); run<1>("IMAD.WIDE.U32 plain (1024 thr/SM)", 2); }
