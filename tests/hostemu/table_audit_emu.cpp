// table_audit_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of hs_table_audit's per-entry checks: a comb table built by
// comb_build_block, and the checks k_table_audit runs over it, in its (window, entry) order.  tests/test_table_audit.py compiles it with
// g++ beside hostemu.cpp; never linked into the product library.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../hotstuff_b200/csrc/verify_core.cuh"

// enc == nullptr: the base point B; otherwise the key's -A, as registration builds it (audit_anchor_point)
static uint32_t anchor(ge_ext &P, const uint8_t *enc) {
  uint32_t w[8];
  if (enc) memcpy(w, enc, 32);
  return audit_anchor_point(P, enc ? w : nullptr);
}

extern "C" {
uint64_t emu_comb_table_bytes(int W) { return comb_table_entries(W) * sizeof(ge_niels); }
// Writes P's comb table at window width W into out (emu_comb_table_bytes(W) bytes); returns 0 when enc does not decompress.
int emu_build_comb_table(const uint8_t *enc, int W, uint8_t *out) {
  ge_ext P;
  const uint32_t ok = anchor(P, enc);
  const int entries = 1 << (W - 1), block = 64, windows = sc_ndigits_rt(W);
  std::vector<ge_niels> t((size_t)windows * comb_window_stride(W));
  std::vector<fe> prod(block);
  for (int w = 0; w < windows; w++)
    for (int b = 0; b < entries / block; b++) comb_build_block(t.data(), P, W, w, b * block, block, prod.data());
  memcpy(out, t.data(), t.size() * sizeof(ge_niels));
  return (int)ok;
}
// 1: every entry passes; 0: *out_win / *out_entry name the first that does not (what k_table_audit's atomic minimum keeps).
int emu_table_audit(const uint8_t *table, int W, const uint8_t *enc, int *out_win, int *out_entry) {
  const ge_niels *tab = reinterpret_cast<const ge_niels *>(table);
  const int n_windows = sc_ndigits_rt(W);
  const uint32_t H = 1u << (W - 1);
  ge_ext P;
  anchor(P, enc);
  for (int win = 0; win < n_windows; win++) {
    const ge_niels *wt = tab + (size_t)win * comb_window_stride(W);
    for (uint32_t m = 0; m <= H; m++) {
      uint32_t ok = audit_entry_local(wt[m], m ? wt[m - 1] : wt[0], wt[1], m);
      if (m == 1) ok &= win == 0 ? audit_anchor(wt[1], P) : audit_link(wt[1], wt[-(ptrdiff_t)comb_window_stride(W) + H]);
      if (!ok) {
        *out_win = win;
        *out_entry = (int)m;
        return 0;
      }
    }
  }
  return 1;
}
}
