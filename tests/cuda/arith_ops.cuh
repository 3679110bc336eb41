// arith_ops.cuh — TEST-ONLY: one field operation by op code, shared by the device harness (arith_harness.cu, nvcc: the generated PTX)
// and its host build (tests/hostemu/arith_emu.cpp, g++ with HS_HOST_EMU: the portable C), so both run the same calls of the same inlines.
// op: 0 mul, 1 sqr, 2 add, 3 sub, 4 canon, 5 invert, 6 pow_p58, 7 neg (emu_fe_op's codes); 8 is_zero, 9 eq, 10 is_neg (0 / 1 in word 0);
// 11 sqr_n with the count in b's low word.
#pragma once
#include "../../hotstuff_b200/csrc/verify_core.cuh"

HS_HD void arith_fe_apply(int op, fe &r, const fe &x, const fe &y) {
  fe_set0(r);
  switch (op) {
    case 0: fe_mul(r, x, y); break;
    case 1: fe_sqr(r, x); break;
    case 2: fe_add(r, x, y); break;
    case 3: fe_sub(r, x, y); break;
    case 4: fe_canon(r, x); break;
    case 5: fe_invert(r, x); break;
    case 6: fe_pow_p58(r, x); break;
    case 7: fe_neg(r, x); break;
    case 8: r.v[0] = fe_is_zero(x); break;
    case 9: r.v[0] = fe_eq(x, y); break;
    case 10: r.v[0] = fe_is_neg(x); break;
    case 11: fe_sqr_n(r, x, (int)y.v[0]); break;
    default: break;
  }
}
