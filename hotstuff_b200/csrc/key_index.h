// key_index.h — the key -> slot index of the per-key comb tables: an open-addressing hash table over 32-byte key bytes with linear
// probing.  The host builds it (key_index) and uploads its `slots`; the device probes the same table (key_probe in hs_engine.cu).
// key_hash is the one hash both sides use.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#define HS_NO_KEY 0xffffffffu  // no key slot: an empty hash slot, or a key that is not in the index

#ifdef __CUDACC__
__host__ __device__
#endif
inline uint32_t key_hash(const uint32_t *w) {
  uint32_t h = 0x9e3779b9u;
  for (int i = 0; i < 8; i++) {
    h ^= w[i];
    h *= 0x85ebca6bu;
    h ^= h >> 15;
  }
  return h;
}

// Hash slot -> key slot over a caller's key-bytes array (slot i's key at pks + 32 i).  The capacity is the smallest power of two >= 16
// and >= twice the key slots it is sized for, so a probe always meets an empty hash slot.
struct key_index {
  std::vector<uint32_t> slots;  // HS_NO_KEY = empty
  uint32_t mask = 0;            // capacity - 1

  static uint32_t capacity_for(size_t n_slots) {
    uint32_t cap = 16;
    while (cap < 2 * n_slots) cap <<= 1;
    return cap;
  }
  void reset(size_t n_slots) {  // empty, sized for n_slots key slots
    slots.assign(capacity_for(n_slots), HS_NO_KEY);
    mask = (uint32_t)slots.size() - 1;
  }
  void clear() { std::fill(slots.begin(), slots.end(), HS_NO_KEY); }

  // The first key slot on key's probe path whose bytes equal key and for which accept(slot) holds, else HS_NO_KEY.  accept is asked
  // before the slot's bytes are read, so it may bound the slots pks holds.
  template <class Accept>
  uint32_t find(const uint8_t *pks, const uint8_t *key, Accept accept) const {
    if (slots.empty()) return HS_NO_KEY;
    uint32_t h = home(key);
    for (uint32_t probe = 0; probe <= mask && slots[h] != HS_NO_KEY; probe++, h = (h + 1) & mask)
      if (accept(slots[h]) && memcmp(pks + 32 * (size_t)slots[h], key, 32) == 0) return slots[h];
    return HS_NO_KEY;
  }
  // Inserts key slot idx unless its probe path already holds an accepted slot with the same bytes; returns whether it did.
  template <class Accept = bool (*)(uint32_t)>
  bool insert_absent(const uint8_t *pks, uint32_t idx, Accept accept = any) {
    const uint8_t *key = pks + 32 * (size_t)idx;
    uint32_t h = home(key);
    for (; slots[h] != HS_NO_KEY; h = (h + 1) & mask)
      if (accept(slots[h]) && memcmp(pks + 32 * (size_t)slots[h], key, 32) == 0) return false;
    slots[h] = idx;
    return true;
  }
  // Clears the table, then inserts the key slots 0 .. n-1 for which in_service(i) holds, in index order: of equal key bytes the first
  // wins.  Inserting them one by one with insert_absent in that order gives the same table.
  template <class InService>
  void build(const uint8_t *pks, size_t n, InService in_service) {
    clear();
    for (size_t i = 0; i < n; i++)
      if (in_service(i)) insert_absent(pks, (uint32_t)i);
  }

 private:
  static bool any(uint32_t) { return true; }
  uint32_t home(const uint8_t *key) const {
    uint32_t w[8];
    memcpy(w, key, 32);
    return key_hash(w) & mask;
  }
};
