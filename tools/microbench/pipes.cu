// Instruction-pipe throughput microbenchmark for sm_90a (H100).
// Measures lane-ops / clk / SM for the integer instructions the field arithmetic is built from,
// so the limb representation is chosen from measurement, not folklore.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "device.cuh"

#define ITERS 4096
#define CK(x) do { cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA error %s at %d\n",cudaGetErrorString(e),__LINE__); return 1;} } while(0)

template <int KIND>
__global__ void __launch_bounds__(1024, 1) k(uint32_t *out, unsigned long long *cyc, uint32_t seed) {
  uint32_t a = seed + threadIdx.x, b = seed * 3 + 1;
  uint32_t r0 = a, r1 = a + 1, r2 = a + 2, r3 = a + 3, r4 = a + 4, r5 = a + 5, r6 = a + 6, r7 = a + 7;
  unsigned long long w0 = a, w1 = a + 1, w2 = a + 2, w3 = a + 3, w4 = a + 4, w5 = a + 5, w6 = a + 6, w7 = a + 7;
  double d0 = a, d1 = a + 1, d2 = a + 2, d3 = a + 3, d4 = a + 4, d5 = a + 5, d6 = a + 6, d7 = a + 7, db = 1.0000001;
  __syncthreads();
  unsigned long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < ITERS; i++) {
    if (KIND == 0) {  // IMAD lo
#define OP(r) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(r) : "r"(b), "r"(a));
      OP(r0) OP(r1) OP(r2) OP(r3) OP(r4) OP(r5) OP(r6) OP(r7)
#undef OP
    } else if (KIND == 1) {  // IMAD.WIDE.U32 64-bit accumulate
#define OP(w) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(a), "r"(b));
      OP(w0) OP(w1) OP(w2) OP(w3) OP(w4) OP(w5) OP(w6) OP(w7)
#undef OP
    } else if (KIND == 2) {  // IMAD.HI.U32
#define OP(r) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(r) : "r"(b), "r"(a));
      OP(r0) OP(r1) OP(r2) OP(r3) OP(r4) OP(r5) OP(r6) OP(r7)
#undef OP
    } else if (KIND == 3) {  // IADD3
#define OP(r) asm volatile("add.u32 %0, %0, %1;" : "+r"(r) : "r"(b));
      OP(r0) OP(r1) OP(r2) OP(r3) OP(r4) OP(r5) OP(r6) OP(r7)
#undef OP
    } else if (KIND == 4) {  // carry chain add.cc / addc.cc (8 long)
      asm volatile("add.cc.u32 %0, %0, %8;\n\taddc.cc.u32 %1, %1, %8;\n\taddc.cc.u32 %2, %2, %8;\n\taddc.cc.u32 %3, %3, %8;\n\t"
                   "addc.cc.u32 %4, %4, %8;\n\taddc.cc.u32 %5, %5, %8;\n\taddc.cc.u32 %6, %6, %8;\n\taddc.u32 %7, %7, %8;"
                   : "+r"(r0), "+r"(r1), "+r"(r2), "+r"(r3), "+r"(r4), "+r"(r5), "+r"(r6), "+r"(r7) : "r"(b));
    } else if (KIND == 5) {  // mad.lo.cc + madc.hi.cc pairs (does ptxas fuse to IMAD.WIDE.X?)
      asm volatile("mad.lo.cc.u32 %0, %8, %9, %0;\n\tmadc.hi.cc.u32 %1, %8, %9, %1;\n\t"
                   "madc.lo.cc.u32 %2, %8, %9, %2;\n\tmadc.hi.cc.u32 %3, %8, %9, %3;\n\t"
                   "madc.lo.cc.u32 %4, %8, %9, %4;\n\tmadc.hi.cc.u32 %5, %8, %9, %5;\n\t"
                   "madc.lo.cc.u32 %6, %8, %9, %6;\n\tmadc.hi.u32 %7, %8, %9, %7;"
                   : "+r"(r0), "+r"(r1), "+r"(r2), "+r"(r3), "+r"(r4), "+r"(r5), "+r"(r6), "+r"(r7) : "r"(a), "r"(b));
    } else if (KIND == 6) {  // LOP3
#define OP(r) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(r) : "r"(b), "r"(a));
      OP(r0) OP(r1) OP(r2) OP(r3) OP(r4) OP(r5) OP(r6) OP(r7)
#undef OP
    } else if (KIND == 7) {  // SHF funnel shift
#define OP(r) asm volatile("shf.l.wrap.b32 %0, %0, %1, 7;" : "+r"(r) : "r"(b));
      OP(r0) OP(r1) OP(r2) OP(r3) OP(r4) OP(r5) OP(r6) OP(r7)
#undef OP
    } else if (KIND == 8) {  // DFMA
#define OP(d) asm volatile("fma.rn.f64 %0, %0, %1, %1;" : "+d"(d) : "d"(db));
      OP(d0) OP(d1) OP(d2) OP(d3) OP(d4) OP(d5) OP(d6) OP(d7)
#undef OP
    } else if (KIND == 9) {  // 4 IMAD.WIDE + 4 IADD3 interleaved (dual-pipe issue?)
#define OPW(w) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(a), "r"(b));
#define OPA(r) asm volatile("add.u32 %0, %0, %1;" : "+r"(r) : "r"(b));
      OPW(w0) OPA(r0) OPW(w1) OPA(r1) OPW(w2) OPA(r2) OPW(w3) OPA(r3)
#undef OPW
#undef OPA
    } else if (KIND == 10) {  // 4 IMAD lo + 4 IADD3 interleaved
#define OPW(r) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(r) : "r"(b), "r"(a));
#define OPA(r) asm volatile("add.u32 %0, %0, %1;" : "+r"(r) : "r"(b));
      OPW(r4) OPA(r0) OPW(r5) OPA(r1) OPW(r6) OPA(r2) OPW(r7) OPA(r3)
#undef OPW
#undef OPA
    } else if (KIND == 11) {  // 4 IMAD.WIDE + 4 DFMA interleaved (separate fp64 pipe?)
#define OPW(w) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w) : "r"(a), "r"(b));
#define OPD(d) asm volatile("fma.rn.f64 %0, %0, %1, %1;" : "+d"(d) : "d"(db));
      OPW(w0) OPD(d0) OPW(w1) OPD(d1) OPW(w2) OPD(d2) OPW(w3) OPD(d3)
#undef OPW
#undef OPD
    } else if (KIND == 12) {  // mul.wide.u32 (no accumulate)
#define OP(w, r) asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(w) : "r"(r), "r"(b)); r ^= (uint32_t)w;
      OP(w0, r0) OP(w1, r1) OP(w2, r2) OP(w3, r3) OP(w4, r4) OP(w5, r5) OP(w6, r6) OP(w7, r7)
#undef OP
    } else if (KIND == 13) {  // 64-bit add (IADD3 + IADD3.X)
#define OP(w) asm volatile("add.u64 %0, %0, %1;" : "+l"(w) : "l"(w7));
      OP(w0) OP(w1) OP(w2) OP(w3) OP(w4) OP(w5) OP(w6) OP(w0)
#undef OP
    }
  }
  unsigned long long t1 = clock64();
  uint32_t acc = r0 ^ r1 ^ r2 ^ r3 ^ r4 ^ r5 ^ r6 ^ r7;
  unsigned long long wacc = w0 ^ w1 ^ w2 ^ w3 ^ w4 ^ w5 ^ w6 ^ w7;
  double dacc = d0 + d1 + d2 + d3 + d4 + d5 + d6 + d7;
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc ^ (uint32_t)wacc ^ (uint32_t)(wacc >> 32) ^ (uint32_t)dacc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int KIND>
int run(const char *name, int threads) {
  uint32_t *out; unsigned long long *cyc;
  int blocks = dev_sms();
  CK(cudaMalloc(&out, blocks * 1024 * 4)); CK(cudaMalloc(&cyc, blocks * 8));
  k<KIND><<<blocks, threads>>>(out, cyc, 12345);  // warm-up
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<KIND><<<blocks, threads>>>(out, cyc, 12345);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  unsigned long long h[1024]; CK(cudaMemcpy(h, cyc, blocks * sizeof(h[0]), cudaMemcpyDeviceToHost));
  double avg = 0; for (int i = 0; i < blocks; i++) avg += (double)h[i]; avg /= blocks;
  double ops = (double)ITERS * 8.0 * threads;  // PTX-level ops per SM (block)
  printf("%-34s threads=%4d  cycles=%9.0f  ptx-ops/clk/SM=%7.2f  ms=%.3f  (eff MHz=%.0f)\n", name, threads, avg, ops / avg, ms, avg / ms / 1e3);
  cudaFree(out); cudaFree(cyc);
  return 0;
}

int main() {
  for (int threads : {256, 512, 1024}) {
    run<0>("IMAD lo", threads);
    run<1>("IMAD.WIDE.U32 acc64", threads);
    run<2>("IMAD.HI.U32", threads);
    run<3>("IADD (add.u32)", threads);
    run<4>("add.cc/addc chain x8", threads);
    run<5>("mad.lo.cc/madc.hi.cc chain x8", threads);
    run<6>("LOP3", threads);
    run<7>("SHF", threads);
    run<8>("DFMA", threads);
    run<9>("4 IMAD.WIDE + 4 IADD mix", threads);
    run<10>("4 IMAD.lo + 4 IADD mix", threads);
    run<11>("4 IMAD.WIDE + 4 DFMA mix", threads);
    run<12>("mul.wide.u32 (+xor)", threads);
    run<13>("add.u64", threads);
  }
  return 0;
}
