// table_mend_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of hs_table_mend's two device steps: the window findings the WINDOWS form
// of k_table_audit reports (audit_mend_flags over the checks it runs, in its order), and the per-block recomputation k_mend_windows
// runs (comb_mend_block).  tests/test_table_mend_emu.py compiles it with g++; never linked into the product library.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>
#include "../../hotstuff_b200/csrc/verify_core.cuh"

// enc == nullptr: the base point B; otherwise the key's -A (audit_anchor_point, as k_mend_windows takes it)
static uint32_t anchor(ge_ext &P, const uint8_t *enc) {
  uint32_t w[8];
  if (enc) memcpy(w, enc, 32);
  return audit_anchor_point(P, enc ? w : nullptr);
}

extern "C" {
uint64_t emu_comb_table_bytes(int W) { return comb_table_entries(W) * sizeof(ge_niels); }
int emu_comb_windows(int W) { return sc_ndigits_rt(W); }
// P's comb table at window width W, built by comb_build_block as k_build_comb builds it.
int emu_build_comb_table(const uint8_t *enc, int W, uint8_t *out) {
  ge_ext P;
  const uint32_t ok = anchor(P, enc);
  const int entries = 1 << (W - 1), windows = sc_ndigits_rt(W);
  std::vector<fe> prod(64);
  ge_niels *t = reinterpret_cast<ge_niels *>(out);
  for (int w = 0; w < windows; w++)
    for (int b = 0; b < entries / 64; b++) comb_build_block(t, P, W, w, b * 64, 64, prod.data());
  return (int)ok;
}
// The window findings of the table's audit: out[i] = 1 for each flagged window i, out[windows] = 1 when the anchor failed.
void emu_mend_windows(const uint8_t *table, int W, const uint8_t *enc, uint8_t *out) {
  const ge_niels *tab = reinterpret_cast<const ge_niels *>(table);
  const int n_windows = sc_ndigits_rt(W);
  const uint32_t H = 1u << (W - 1);
  ge_ext P;
  anchor(P, enc);
  memset(out, 0, n_windows + 1);
  for (int win = 0; win < n_windows; win++) {
    const ge_niels *wt = tab + (size_t)win * comb_window_stride(W);
    for (uint32_t m = 0; m <= H; m++) {
      const uint32_t ok = audit_entry_local(wt[m], m ? wt[m - 1] : wt[0], wt[1], m);
      const uint32_t edge = m != 1 ? 1u : win == 0 ? audit_anchor(wt[1], P) : audit_link(wt[1], wt[-(ptrdiff_t)comb_window_stride(W) + H]);
      const uint32_t f = audit_mend_flags(win, m, ok, edge);
      if (f & 1u) out[win] = 1;
      if (f & 2u) out[win - 1] = 1;
      if (f & 4u) out[n_windows] = 1;
    }
  }
}
// k_mend_windows' work on window `win` of the table, every block of it: returns the entries it stored.
uint64_t emu_mend_window(uint8_t *table, int W, const uint8_t *enc, int win) {
  ge_ext P;
  if (!anchor(P, enc)) return 0;
  const int entries = 1 << (W - 1);
  std::vector<ge_niels> stage(65);
  std::vector<fe> prod(64);
  ge_niels *window = reinterpret_cast<ge_niels *>(table) + (size_t)win * comb_window_stride(W);
  uint64_t stored = 0;
  for (int b = 0; b < entries / 64; b++) stored += comb_mend_block(window, stage.data(), P, W, win, b * 64, 64, prod.data());
  return stored;
}
// One block of window `win` at any width (the 24-bit tables are too large to build on a CPU): the mend's entries first .. first + 64
// (entry first only for first == 0) stored into `mended` over zeros, and comb_build_block's into `built`, each 65 entries; returns
// the mend's count of stored entries.
uint64_t emu_mend_block(const uint8_t *enc, int W, int win, int first, uint8_t *mended, uint8_t *built) {
  ge_ext P;
  anchor(P, enc);
  std::vector<ge_niels> stage(65);
  std::vector<fe> prod(64);
  ge_niels *m = reinterpret_cast<ge_niels *>(mended), *b = reinterpret_cast<ge_niels *>(built);
  memset(m, 0, 65 * sizeof(ge_niels));
  const uint64_t n = comb_mend_block(m - first, stage.data(), P, W, win, first, 64, prod.data());
  comb_build_block(b - (size_t)win * comb_window_stride(W) - first, P, W, win, first, 64, prod.data());
  return n;
}
}
