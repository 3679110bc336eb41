// explain_select_emu.cpp — TEST-ONLY host build (HS_HOST_EMU) of hs_explain_groups_dev's selection: the per-word zero bits, the ranks the
// kernels compute (block sums of HS_SEL_WORDS words, their exclusive offsets, each word's exclusive rank within its block) and the
// ordered scatter, with the helpers of explain_select.cuh.  tests/test_explain_dev.py compiles it with g++; never linked into the product
// library.
#include <cstddef>
#include <cstdint>
#include <vector>
#include "../../hotstuff_b200/csrc/explain_select.cuh"

extern "C" {
// The selection over a bitmap of n items with max_explain = max_explain: list receives the examined indices, out the kernels' first two
// words ([0] zero bits, [1] items examined).
void emu_select(const uint32_t *bm, uint64_t n, uint64_t max_explain, uint32_t *list, uint32_t *out) {
  const uint64_t n_words = (n + 31) / 32, n_blocks = (n_words + HS_SEL_WORDS - 1) / HS_SEL_WORDS;
  const uint64_t cap = max_explain && max_explain < n ? max_explain : n;
  std::vector<uint32_t> boff(n_blocks);
  uint32_t carry = 0;
  for (uint64_t b = 0; b < n_blocks; b++) {  // k_sel_count, then k_sel_top's exclusive offsets
    boff[b] = carry;
    for (uint64_t w = b * HS_SEL_WORDS; w < n_words && w < (b + 1) * HS_SEL_WORDS; w++) carry += __builtin_popcount(bitmap_zero_bits(bm[w], n, w));
  }
  out[0] = carry;
  out[1] = cap < carry ? (uint32_t)cap : carry;
  for (uint64_t b = 0; b < n_blocks; b++) {  // k_sel_scatter
    uint32_t r = 0;
    for (uint64_t w = b * HS_SEL_WORDS; w < n_words && w < (b + 1) * HS_SEL_WORDS; w++) {
      const uint32_t zeros = bitmap_zero_bits(bm[w], n, w);
      select_scatter(zeros, (uint64_t)boff[b] + r, w, out[1], list);
      r += __builtin_popcount(zeros);
    }
  }
}
uint32_t emu_valid_in_mode(uint32_t why, uint32_t mode_byte) { return why_valid_in_mode(why, mode_byte); }
}
