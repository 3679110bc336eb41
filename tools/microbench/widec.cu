// Cost of the carry-out-only wide mad (IMAD.WIDE.U32 Rd, Pc, ...) + a separate IADD3.X carry counter,
// versus the carry-in/out form (.X).  Decides whether deferred-carry accumulation beats the .X chains.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"
#define ITERS 4096
template <int KIND>
__global__ void __launch_bounds__(512, 1) k(uint32_t *out, uint32_t seed) {
  uint32_t x = seed + threadIdx.x, y = seed * 3 + threadIdx.x * 7 + 1;
  uint32_t l0 = x, h0 = y, l1 = x + 1, h1 = y + 1, l2 = x + 2, h2 = y + 2, l3 = x + 3, h3 = y + 3;
  uint32_t l4 = x + 4, h4 = y + 4, l5 = x + 5, h5 = y + 5, l6 = x + 6, h6 = y + 6, l7 = x + 7, h7 = y + 7;
  uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0, c6 = 0, c7 = 0;
#pragma unroll 1
  for (int i = 0; i < ITERS; i++) {
    if (KIND == 0) {  // 8 x (wide mad with carry-out, carry counted in a separate register)
#define OP(l, h, c) asm volatile("mad.lo.cc.u32 %0, %3, %4, %0;\n\tmadc.hi.cc.u32 %1, %3, %4, %1;\n\taddc.u32 %2, %2, 0;" : "+r"(l), "+r"(h), "+r"(c) : "r"(x), "r"(y));
      OP(l0, h0, c0) OP(l1, h1, c1) OP(l2, h2, c2) OP(l3, h3, c3) OP(l4, h4, c4) OP(l5, h5, c5) OP(l6, h6, c6) OP(l7, h7, c7)
#undef OP
    } else if (KIND == 1) {  // 8 plain wide mads (no carry)
#define OP(l, h) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.u32 %1, %2, %3, %1;" : "+r"(l), "+r"(h) : "r"(x), "r"(y));
      OP(l0, h0) OP(l1, h1) OP(l2, h2) OP(l3, h3) OP(l4, h4) OP(l5, h5) OP(l6, h6) OP(l7, h7)
#undef OP
    } else if (KIND == 2) {  // two 4-long .X chains
      asm volatile("mad.lo.cc.u32 %0, %8, %9, %0;\n\tmadc.hi.cc.u32 %1, %8, %9, %1;\n\tmadc.lo.cc.u32 %2, %8, %9, %2;\n\tmadc.hi.cc.u32 %3, %8, %9, %3;\n\t"
                   "madc.lo.cc.u32 %4, %8, %9, %4;\n\tmadc.hi.cc.u32 %5, %8, %9, %5;\n\tmadc.lo.cc.u32 %6, %8, %9, %6;\n\tmadc.hi.u32 %7, %8, %9, %7;"
                   : "+r"(l0), "+r"(h0), "+r"(l1), "+r"(h1), "+r"(l2), "+r"(h2), "+r"(l3), "+r"(h3) : "r"(x), "r"(y));
      asm volatile("mad.lo.cc.u32 %0, %8, %9, %0;\n\tmadc.hi.cc.u32 %1, %8, %9, %1;\n\tmadc.lo.cc.u32 %2, %8, %9, %2;\n\tmadc.hi.cc.u32 %3, %8, %9, %3;\n\t"
                   "madc.lo.cc.u32 %4, %8, %9, %4;\n\tmadc.hi.cc.u32 %5, %8, %9, %5;\n\tmadc.lo.cc.u32 %6, %8, %9, %6;\n\tmadc.hi.u32 %7, %8, %9, %7;"
                   : "+r"(l4), "+r"(h4), "+r"(l5), "+r"(h5), "+r"(l6), "+r"(h6), "+r"(l7), "+r"(h7) : "r"(y), "r"(x));
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = l0 ^ h0 ^ l1 ^ h1 ^ l2 ^ h2 ^ l3 ^ h3 ^ l4 ^ h4 ^ l5 ^ h5 ^ l6 ^ h6 ^ l7 ^ h7 ^ c0 ^ c1 ^ c2 ^ c3 ^ c4 ^ c5 ^ c6 ^ c7;
}
template <int KIND> void run(const char *name) {
  uint32_t *out; int blocks = dev_sms() * 2, threads = 512;
  cudaMalloc(&out, blocks * threads * 4);
  k<KIND><<<blocks, threads>>>(out, 12345); cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0); k<KIND><<<blocks, threads>>>(out, 12345); cudaEventRecord(e1); cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  printf("%-44s %.3f ms  wide-mads/clk/SM = %.2f (at the maximum SM clock)\n", name, ms, (double)ITERS * 8.0 * threads * 2 / (ms * 1e-3 * dev_clock_hz()));
  cudaFree(out);
}
int main() { run<0>("carry-out wide mad + IADD3.X counter"); run<1>("plain wide mad"); run<2>(".X chains (4 long)"); }
