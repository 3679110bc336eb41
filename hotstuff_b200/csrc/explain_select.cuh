// explain_select.cuh — the index arithmetic of hs_explain_groups_dev: which items of a pass it examines, and which of them are engine
// faults.  Shared by the kernels in hs_engine.cu and the host emulation (tests/hostemu/explain_select_emu.cpp).
//
// The selection is the lowest-index `cap` items whose bit is 0: word w of the bitmap contributes the zero bits of its valid items
// (bitmap_zero_bits), the words are ranked by an exclusive prefix sum of those counts, and a word whose rank is below cap writes its
// items' indices, in increasing order, to list[rank ..] until the list holds cap (select_scatter).
#pragma once
#include <cstdint>
#include "../../include/hs_crypto.h"
#include "fe.cuh"  // HS_HD

#define HS_SEL_WORDS 256  // bitmap words per block of the selection kernels (8,192 items)

// The zero bits of word w of a bitmap over n items (the unused high bits of the last word count as ones).
HS_HD uint32_t bitmap_zero_bits(uint32_t word, uint64_t n, uint64_t w) {
  const uint32_t valid = ((n & 31) && w == (n - 1) / 32) ? ((1u << (n & 31)) - 1u) : 0xffffffffu;
  return ~word & valid;
}

// Writes the item index of every set bit of `zeros` (word w), lowest first, to list[rank], list[rank + 1], .. while the index into the
// list is below cap.
HS_HD void select_scatter(uint32_t zeros, uint64_t rank, uint64_t w, uint64_t cap, uint32_t *list) {
  for (; zeros && rank < cap; zeros &= zeros - 1, rank++) {
#if defined(__CUDA_ARCH__)
    const uint32_t b = (uint32_t)__ffs(zeros) - 1;
#else
    const uint32_t b = (uint32_t)__builtin_ctz(zeros);
#endif
    list[rank] = (uint32_t)(w * 32 + b);
  }
}

// A rejected item is an engine fault when its table-free mask says it is valid in its mode: mode byte 1 (HS_MODE_BATCH_EQ) allows
// only the small-order bits, and every other byte is strict, as hs_verify_groups_dev judges it.
HS_HD bool why_valid_in_mode(uint32_t why, uint32_t mode_byte) {
  return mode_byte == HS_MODE_BATCH_EQ ? (why & ~(uint32_t)(HS_WHY_A_SMALL | HS_WHY_R_SMALL)) == 0 : why == 0;
}
