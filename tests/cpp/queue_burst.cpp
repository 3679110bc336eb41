// Verify-queue burst driver (tests/test_queue.py): native threads submit single-record requests to ONE hs_queue as fast as
// they can, then every ticket is read and checked against the expected verdicts; prints the queue launches the burst took.
//   input file: u32 n_keys | n_keys x 32 key bytes (registered as the committee) | u32 n | n x hs_rec128 | n expected verdicts (0/1)
//   queue_burst FILE THREADS        burst through the C ABI (hs_queue_submit from THREADS threads, then hs_queue_wait per ticket)
//   queue_burst FILE THREADS --hpp  the same records through hs::VerifyQueue (std::future per request)
// Prints one JSON line; exit status 0 only if every verdict matched.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <thread>
#include <vector>

#include "../../include/hs_crypto.hpp"

static uint32_t rd32(const std::vector<uint8_t> &b, size_t &o) {
  uint32_t v;
  memcpy(&v, b.data() + o, 4);
  o += 4;
  return v;
}

int main(int argc, char **argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: queue_burst FILE THREADS [--hpp]\n");
    return 2;
  }
  std::ifstream f(argv[1], std::ios::binary);
  std::vector<uint8_t> blob((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  const int nth = atoi(argv[2]);
  const bool hpp = argc > 3 && strcmp(argv[3], "--hpp") == 0;
  size_t o = 0;
  const uint32_t n_keys = rd32(blob, o);
  const uint8_t *keys = blob.data() + o;
  o += (size_t)n_keys * 32;
  const uint32_t n = rd32(blob, o);
  std::vector<hs_rec128> recs(n);
  memcpy(recs.data(), blob.data() + o, (size_t)n * sizeof(hs_rec128));
  o += (size_t)n * sizeof(hs_rec128);
  const uint8_t *want = blob.data() + o;

  hs::Engine e(0);
  std::vector<uint32_t> valid((n_keys + 31) / 32);
  e.check(hs_committee_register(e.raw(), keys, n_keys, valid.data()), "hs_committee_register");
  std::atomic<int> bad{0}, full{0};
  std::atomic<int> go{0};
  uint64_t launches = 0;
  if (!hpp) {
    hs_queue *q = nullptr;
    e.check(hs_queue_create(e.raw(), 0, &q), "hs_queue_create");
    std::vector<size_t> ticket(n);
    const uint64_t l0 = hs_kernel_launches(e.raw());
    std::vector<std::thread> ts;
    for (int t = 0; t < nth; t++)
      ts.emplace_back([&, t] {
        while (!go.load()) {
        }
        for (size_t i = t; i < n; i += nth) {
          int rc;
          while ((rc = hs_queue_submit(q, &recs[i], 1, HS_MODE_STRICT, nullptr, nullptr, &ticket[i])) == HS_ERR_NOMEM) {
            full++;
            std::this_thread::yield();
          }
          if (rc != HS_OK) bad++;
        }
      });
    go = 1;
    for (auto &t : ts) t.join();
    for (size_t i = 0; i < n; i++) {
      uint32_t bm = 0;
      if (hs_queue_wait(q, ticket[i], &bm) != HS_OK || (bm & 1u) != want[i]) bad++;
    }
    launches = hs_kernel_launches(e.raw()) - l0;
    uint32_t bm = 0;
    if (hs_queue_wait(q, ticket[0], &bm) != HS_ERR_ARG) bad++;  // a ticket is read once
    hs_queue_destroy(q);
  } else {
    hs::VerifyQueue vq(e);
    std::vector<std::future<std::vector<bool>>> fut(n);
    const uint64_t l0 = hs_kernel_launches(e.raw());
    std::vector<std::thread> ts;
    for (int t = 0; t < nth; t++)
      ts.emplace_back([&, t] {
        while (!go.load()) {
        }
        for (size_t i = t; i < n; i += nth) {
          for (;;) {
            try {
              fut[i] = vq.submit(&recs[i], 1);
              break;
            } catch (const hs::QueueFull &) {
              full++;
              std::this_thread::yield();
            }
          }
        }
      });
    go = 1;
    for (auto &t : ts) t.join();
    for (size_t i = 0; i < n; i++) {
      std::vector<bool> v = fut[i].get();
      if (v.size() != 1 || (uint8_t)v[0] != want[i]) bad++;
    }
    launches = hs_kernel_launches(e.raw()) - l0;
  }
  printf("{\"records\": %u, \"threads\": %d, \"queue_launches\": %llu, \"records_per_launch\": %.2f, \"ring_full_retries\": %d, \"mismatches\": %d}\n", n, nth,
         (unsigned long long)launches, launches ? (double)n / (double)launches : 0.0, full.load(), bad.load());
  return bad.load() ? 1 : 0;
}
