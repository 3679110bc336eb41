// key_index_emu.cpp — TEST-ONLY host build of key_index.h, the key -> slot index the engine builds on the host and uploads for
// k_key_lookup.  tests/test_key_index.py compiles it with g++; never linked into the product library.
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include "../../hotstuff_b200/csrc/key_index.h"

static key_index view(const uint32_t *slots, uint32_t cap) {
  key_index ix;
  ix.slots.assign(slots, slots + cap);
  ix.mask = cap - 1;
  return ix;
}

extern "C" {
uint32_t emu_capacity(size_t n_slots) { return key_index::capacity_for(n_slots); }
// The table build() makes over pks[0 .. n) with in_service[i] != 0, sized for n_slots key slots (emu_capacity(n_slots) words).
void emu_build(const uint8_t *pks, size_t n, size_t n_slots, const uint8_t *in_service, uint32_t *out) {
  key_index ix;
  ix.reset(n_slots);
  ix.build(pks, n, [&](size_t i) { return in_service[i] != 0; });
  std::copy(ix.slots.begin(), ix.slots.end(), out);
}
// find() of keys[0 .. m) in the table `slots` of cap words, accepting a slot idx < bound, or accepted[idx] != 0 when accepted != NULL.
void emu_find(const uint32_t *slots, uint32_t cap, const uint8_t *pks, const uint8_t *keys, size_t m, uint32_t bound, const uint8_t *accepted,
              uint32_t *out) {
  const key_index ix = view(slots, cap);
  for (size_t k = 0; k < m; k++)
    out[k] = accepted ? ix.find(pks, keys + 32 * k, [&](uint32_t idx) { return accepted[idx] != 0; })
                      : ix.find(pks, keys + 32 * k, [&](uint32_t idx) { return idx < bound; });
}
// insert_absent() of slots idx[0 .. m) in order into the table `slots` of cap words (updated in place), accepting every slot, or a slot
// with accepted[slot] != 0 when accepted != NULL; inserted[k] = its result.
void emu_insert_absent(uint32_t *slots, uint32_t cap, const uint8_t *pks, const uint32_t *idx, size_t m, const uint8_t *accepted,
                       uint8_t *inserted) {
  key_index ix = view(slots, cap);
  for (size_t k = 0; k < m; k++)
    inserted[k] = accepted ? ix.insert_absent(pks, idx[k], [&](uint32_t s) { return accepted[s] != 0; }) : ix.insert_absent(pks, idx[k]);
  std::copy(ix.slots.begin(), ix.slots.end(), slots);
}
}
