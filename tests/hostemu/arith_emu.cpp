// arith_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of the field operations the device harness runs (tests/cuda/arith_ops.cuh), with the
// portable C in place of the generated PTX.  tests/test_device_arith_edges.py compiles it with g++; never linked into the product library.
#include <cstdint>
#include <cstring>
#include "../cuda/arith_ops.cuh"

extern "C" {
// a, b, out: n field elements of 8 little-endian words each
void emu_arith_fe_op(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, int n) {
  for (int i = 0; i < n; i++) {
    fe x, y, r;
    memcpy(x.v, a + 8 * i, 32);
    memcpy(y.v, b + 8 * i, 32);
    arith_fe_apply(op, r, x, y);
    memcpy(out + 8 * i, r.v, 32);
  }
}
}
