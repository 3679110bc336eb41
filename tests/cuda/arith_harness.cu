// arith_harness.cu — TEST-ONLY: the device field and scalar primitives, one thread per input, behind host-array wrappers.
// It includes the same headers as the verify kernels, so fe_* runs the generated PTX (fe_asm.cuh) and sc_* the same inlines; the
// host build of the field operations (tests/hostemu/arith_emu.cpp) runs the portable C of the same headers through the same op table.
// Built by tests/test_device_arith_edges.py into a temporary directory; never linked into the product library.
#include <cuda_runtime.h>
#include <cstdint>
#include "arith_ops.cuh"

// one thread per element: out[i] = op(a[i], b[i]) (op codes: arith_ops.cuh)
__global__ void k_fe_op(int op, const fe *a, const fe *b, fe *out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const fe x = a[i], y = b[i];
  fe r;
  arith_fe_apply(op, r, x, y);
  out[i] = r;
}

// op 0: sc_reduce512 of 16 input words -> 8 output words; op 1: sc_is_canonical of 8 input words -> word 0;
// op 2: sc_digits_rt(W) of 8 input words -> sc_ndigits_rt(W) signed digits.  Each item reads 16 and writes 64 words.
#define ARITH_SC_OUT 64
__global__ void k_sc_op(int op, int W, const uint32_t *in, int32_t *out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t *x = in + 16 * (size_t)i;
  int32_t *o = out + ARITH_SC_OUT * (size_t)i;
  uint32_t s[8];
  for (int j = 0; j < 8; j++) s[j] = x[j];
  if (op == 0) {
    uint32_t w[16], r[8];
    for (int j = 0; j < 16; j++) w[j] = x[j];
    sc_reduce512(r, w);
    for (int j = 0; j < 8; j++) o[j] = (int32_t)r[j];
  } else if (op == 1) {
    o[0] = (int32_t)sc_is_canonical(s);
  } else {
    uint32_t bias[9];
    sc_bias_rt(bias, W);
    sc_digits_rt(o, 1, s, bias, W, sc_ndigits_rt(W));
  }
}

namespace {
// device copies of the wrappers' host arrays, all released when the call returns
struct dev_arrays {
  void *p[3] = {nullptr, nullptr, nullptr};
  ~dev_arrays() {
    for (void *q : p) cudaFree(q);
  }
};
cudaError_t finish(cudaError_t e) { return e != cudaSuccess ? e : cudaDeviceSynchronize(); }
}  // namespace

// a, b, out: n field elements of 8 little-endian words each.  Returns the first CUDA error (cudaSuccess = 0).
extern "C" int arith_fe_op(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, int n) {
  if (n <= 0) return (int)cudaErrorInvalidValue;
  const size_t bytes = (size_t)n * sizeof(fe);
  dev_arrays d;
  cudaError_t e;
  for (int k = 0; k < 3; k++)
    if ((e = cudaMalloc(&d.p[k], bytes)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpy(d.p[0], a, bytes, cudaMemcpyHostToDevice)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpy(d.p[1], b, bytes, cudaMemcpyHostToDevice)) != cudaSuccess) return (int)e;
  k_fe_op<<<(n + 127) / 128, 128>>>(op, (const fe *)d.p[0], (const fe *)d.p[1], (fe *)d.p[2], n);
  if ((e = finish(cudaGetLastError())) != cudaSuccess) return (int)e;
  return (int)cudaMemcpy(out, d.p[2], bytes, cudaMemcpyDeviceToHost);
}

// in: n items of 16 words; out: n items of 64 int32 (see k_sc_op).  W: window width for op 2 (8 .. 26).
extern "C" int arith_sc_op(int op, int W, const uint32_t *in, int32_t *out, int n) {
  if (n <= 0 || (op == 2 && (W < 8 || W > 26))) return (int)cudaErrorInvalidValue;
  dev_arrays d;
  cudaError_t e;
  if ((e = cudaMalloc(&d.p[0], (size_t)n * 16 * 4)) != cudaSuccess) return (int)e;
  if ((e = cudaMalloc(&d.p[1], (size_t)n * ARITH_SC_OUT * 4)) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpy(d.p[0], in, (size_t)n * 16 * 4, cudaMemcpyHostToDevice)) != cudaSuccess) return (int)e;
  if ((e = cudaMemset(d.p[1], 0, (size_t)n * ARITH_SC_OUT * 4)) != cudaSuccess) return (int)e;
  k_sc_op<<<(n + 127) / 128, 128>>>(op, W, (const uint32_t *)d.p[0], (int32_t *)d.p[1], n);
  if ((e = finish(cudaGetLastError())) != cudaSuccess) return (int)e;
  return (int)cudaMemcpy(out, d.p[1], (size_t)n * ARITH_SC_OUT * 4, cudaMemcpyDeviceToHost);
}
