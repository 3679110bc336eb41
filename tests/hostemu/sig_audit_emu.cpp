// sig_audit_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of the signature-cache audit's decision: flags_from_why(explain_record(..)),
// the flag byte k_sig_audit derives for a stored record.  tests/test_sig_audit_flags.py compiles it with g++; never linked into the
// product library.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include "../../hotstuff_b200/csrc/verify_core.cuh"

extern "C" {
uint32_t emu_flags_from_why(uint32_t why) { return flags_from_why(why); }
// out_flags[i] = flags_from_why(explain_record(..)) of record i: sig[i] (R || S), pk[i] and h[i] = SHA-512(R || A || msg).
void emu_audit_flags(const uint8_t *sig, const uint8_t *pk, const uint8_t *h, size_t n, uint8_t *out_flags) {
  for (size_t i = 0; i < n; i++) {
    uint32_t R[8], S[8], A[8], hw[16];
    memcpy(R, sig + 64 * i, 32);
    memcpy(S, sig + 64 * i + 32, 32);
    memcpy(A, pk + 32 * i, 32);
    memcpy(hw, h + 64 * i, 64);
    ge_cached tab[9];
    out_flags[i] = (uint8_t)flags_from_why(explain_record(R, S, A, hw, tab));
  }
}
}
