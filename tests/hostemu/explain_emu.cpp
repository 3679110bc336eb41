// explain_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of explain_record, the table-free per-check decision that k_explain runs for
// hs_explain_rec128.  tests/test_explain.py compiles it with g++; never linked into the product library.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include "../../hotstuff_b200/csrc/verify_core.cuh"

extern "C" {
// out_why[i] = explain_record of record i: sig[i] (64 bytes: R || S), pk[i] (32 bytes) and h[i] = SHA-512(R || A || msg) (64 bytes).
void emu_explain(const uint8_t *sig, const uint8_t *pk, const uint8_t *h, size_t n, uint8_t *out_why) {
  for (size_t i = 0; i < n; i++) {
    uint32_t R[8], S[8], A[8], hw[16];
    memcpy(R, sig + 64 * i, 32);
    memcpy(S, sig + 64 * i + 32, 32);
    memcpy(A, pk + 32 * i, 32);
    memcpy(hw, h + 64 * i, 64);
    ge_cached tab[9];
    out_why[i] = (uint8_t)explain_record(R, S, A, hw, tab);
  }
}
}
