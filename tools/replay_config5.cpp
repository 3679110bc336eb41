// replay_config5.cpp — BASELINE config[4] substitute (SURVEY §8d "Config 5"), C++ against the C ABI.
//
// The Rust node cannot be built here (no cargo), so this REPLAYS the per-node crypto call stream of `fab local`
// (benchmark/fabfile.py:14-33 at 50,000 tx/s, 512 B tx, 4 nodes, 15,000 B batches) and reports per-call latency:
//   per second : ~1,707 Digest calls over ~15.3 kB serialized batches            (mempool/src/processor.rs:30)
//   per round  : 1 strict verify                      (Block::verify, consensus/src/messages.rs:64)
//                1 verify_batch of 3 votes            (QC::verify,    messages.rs:197)
//                3 strict verifies at the leader      (Vote::verify,  messages.rs:144)
// Timed with steady_clock around each C-ABI call (host pointers in, verdicts out) — what the Rust shim would see.
// The CPU column times the oracle (the restatement of the reference's dalek path) on one core for the same calls:
// it is the number the shim's CPU/GPU cut-over is chosen against.  This is a replay of the call pattern, NOT a fab run.
//
// Leader vote burst (after the replay): the N - f Vote::verify calls of one round at the leader (N = 4, 100, 1,000), one
// strict verify of a Digest over a 40-byte preimage per vote, 1 % of the votes corrupted, arriving at once from 16 native
// threads (one per connection task).  Three arms: (a) the verify queue (hs_queue_submit + callback), (b) one synchronous
// hs_verify_rec128(n = 1) per vote from the same 16 threads, (c) the CPU oracle verifying the votes serially on one core (what
// Core does today).  Per-vote latency = burst start -> that vote's verdict; every verdict is checked against the oracle.
//
// Replica block (after the burst): one Block::verify certificate = 1 strict author signature + N - f batch-eq QC votes, 1 % of
// the records corrupted, N = 4 .. 10,000, on a 16,384-record ring.  Three arms per block: (a) one hs_queue_submit_group consumed by
// hs_queue_wait, (b) the synchronous calls the shim makes today (a strict author verify + hs_verify_batch_shared_msg), (c) the CPU
// oracle on one core.  Block during a burst: the N-validator vote burst above (N = 1,000 and 10,000) with one Block certificate
// (668 / 6,668 records) submitted once half the votes are in, (a) through the same queue or (b) as the synchronous calls from
// another thread.  Every queue section prints the queue's counters (hs_queue_stats): which kernel carried how many records.
//
// Certificate preimages (last; alone with argv[3] = certificate_preimages): a TC and a Block with a TC, N = 4 .. 750, verified
// (a) by hashing the preimages on the caller's thread then hs_queue_submit_group, (b) by hs_queue_submit_msgs (the GPU hashes them),
// (c) synchronously; latency and the caller thread's CPU time per certificate, plus hs_queue_digest_stats.
//
// TC after Timeouts (alone with argv[3] = tc_after_timeouts): N = 100, 1,000 and 4,000 Timeouts through the queue, then the TC made
// of their author signatures and the Block carrying it: synchronous calls vs. the queue without vs. with its signature cache.
// Signature-cache cost (alone with argv[3] = sig_cache_cost): the vote burst and replica_block sections with the cache off, then on.
//
// View change (last; alone with argv[3] = view_change): N = 100, 1,000 and 4,000 Timeouts released at once to 16 threads, nearly all
// carrying the same high_qc, through (a) the queue without its certificate cache (synchronous fallback as the Rust module), (b) the
// queue with it, (c) the synchronous batched calls; burst time, signatures verified and hs_queue_cert_stats.
//
// Foreign keys (alone with argv[3] = foreign_keys): single-record vote bursts with no committee registered, and bursts with one
// request by an unregistered key (1 or 500 records) halfway through, with hs_queue_generic off and on (see run_foreign_keys).
//
// Batch lane (alone with argv[3] = batch_lane): a whole hs_verify_groups pass as one queue request, against hs_queue_submit_msgs and
// the synchronous calls, for a Block alone, a Block during the vote burst and a collected view-change burst (see run_batch_lane).
//
// build: g++ -O2 -std=c++17 -pthread tools/replay_config5.cpp -Iinclude -Ioracle -Lhotstuff_b200 -lhs_crypto -Loracle -lhs_oracle -o tools/replay_config5
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <string>
#include <thread>
#include <vector>

#include "hs_crypto.h"
#include "hs_oracle.h"  // input synthesis (signing) and the CPU column only

using clk = std::chrono::steady_clock;
static double us_since(clk::time_point t0) { return std::chrono::duration<double, std::micro>(clk::now() - t0).count(); }
struct series {
  std::vector<double> v;
  double pct(double p) {
    std::vector<double> s = v;
    std::sort(s.begin(), s.end());
    return s.empty() ? 0 : s[(size_t)(p * (s.size() - 1))];
  }
  double mean() {
    double t = 0;
    for (double x : v) t += x;
    return v.empty() ? 0 : t / v.size();
  }
};
static void emit(const char *name, series &g, series &c, bool last) {
  printf("\"%s\": {\"gpu_p50_us\": %.1f, \"gpu_p99_us\": %.1f, \"gpu_mean_us\": %.1f, \"cpu_oracle_1core_p50_us\": %.1f, \"calls\": %zu}%s", name, g.pct(0.5), g.pct(0.99),
         g.mean(), c.pct(0.5), g.v.size(), last ? "" : ", ");
}

// ---- leader vote burst
struct burst_arm {
  series total, vote;  // burst start -> last verdict; burst start -> each vote's verdict
  uint64_t launches = 0;
  int mismatches = 0;
  void emit(const char *name, int bursts, bool last) {
    printf("\"%s\": {\"burst_p50_us\": %.1f, \"burst_min_us\": %.1f, \"vote_p50_us\": %.1f, \"vote_p99_us\": %.1f, \"launches_per_burst\": %.1f, \"mismatches\": %d}%s", name,
           total.pct(0.5), total.pct(0.0), vote.pct(0.5), vote.pct(0.99), (double)launches / bursts, mismatches, last ? "" : ", ");
  }
};
struct burst_vote {
  clk::time_point t0;
  double *lat;
  int *verdict;
};
static void on_vote(void *user, size_t, int status, const uint32_t *bitmap) {
  burst_vote *v = (burst_vote *)user;
  *v->lat = us_since(v->t0);
  __atomic_store_n(v->verdict, status == HS_OK ? (int)(bitmap[0] & 1u) : -1, __ATOMIC_RELEASE);
}
// Signature-cache entries of the queues the vote burst and replica_block sections create (0 = off, as in the default run; the
// sig_cache_cost section runs them both ways).
static size_t g_sig_entries = 0;
// One committee size: `bursts` timed bursts (+3 warm-up) of N - f votes per arm.
static int vote_burst(hs_ctx *ctx, int N, int bursts, bool last) {
  const int f = (N - 1) / 3, nv = N - f, nth = 16;
  std::vector<uint8_t> seeds((size_t)N * 32), pks((size_t)N * 32);
  for (int i = 0; i < N; i++) {
    for (int j = 0; j < 32; j++) seeds[(size_t)i * 32 + j] = (uint8_t)(29 * i + 5 * j + 7 + (i >> 8));
    hso_keygen(&seeds[(size_t)i * 32], &pks[(size_t)i * 32]);
  }
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, pks.data(), N, valid.data()) != HS_OK) return 1;
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 0, &q) != HS_OK) return 1;
  if (g_sig_entries && hs_queue_sig_cache(q, g_sig_entries) != HS_OK) return 1;
  burst_arm a, b, c;
  std::vector<hs_rec128> recs(nv);
  std::vector<int> want(nv), got(nv);
  std::vector<double> lat(nv);
  std::vector<burst_vote> bv(nv);
  for (int r = 0; r < bursts + 3; r++) {
    const bool timed = r >= 3;
    uint8_t pre[40], d[32];  // Vote::digest = SHA-512(hash || round_le)[..32]
    for (int j = 0; j < 32; j++) pre[j] = (uint8_t)(r * 13 + j);
    const uint64_t round = 1000 + (uint64_t)r;
    memcpy(pre + 32, &round, 8);
    hso_digest32(pre, 40, d);
    for (int i = 0; i < nv; i++) {
      const int k = (i * 7 + r) % N;  // who voted varies per round
      hso_sign(&seeds[(size_t)k * 32], d, 32, recs[i].sig);
      memcpy(recs[i].pk, &pks[(size_t)k * 32], 32);
      memcpy(recs[i].msg, d, 32);
      if ((i * 37 + r * 11) % 100 == 0) recs[i].sig[(i + r) % 64] ^= 0x10;  // 1 % corrupted
    }
    // (c) CPU oracle, one core, serial: the reference verdicts
    auto t0 = clk::now();
    for (int i = 0; i < nv; i++) {
      want[i] = hso_verify_strict(recs[i].sig, recs[i].pk, recs[i].msg, 32);
      lat[i] = us_since(t0);
    }
    if (timed) {
      c.total.v.push_back(us_since(t0));
      c.vote.v.insert(c.vote.v.end(), lat.begin(), lat.end());
    }
    // (a) the queue: 16 threads submit their votes as one burst, verdicts arrive through the callback
    std::atomic<int> go{0}, bad{0};
    std::vector<std::thread> ts;
    uint64_t l0 = hs_kernel_launches(ctx);
    for (int t = 0; t < nth; t++)
      ts.emplace_back([&, t] {
        while (!go.load()) {
        }
        for (int i = t; i < nv; i += nth) {
          bv[i] = burst_vote{t0, &lat[i], &got[i]};
          int rc;
          while ((rc = hs_queue_submit(q, &recs[i], 1, HS_MODE_STRICT, on_vote, &bv[i], nullptr)) == HS_ERR_NOMEM) std::this_thread::yield();
          if (rc != HS_OK) bad++;
        }
      });
    std::fill(got.begin(), got.end(), -2);
    t0 = clk::now();  // the threads read it after `go`
    go = 1;
    for (auto &t : ts) t.join();
    ts.clear();
    for (int i = 0; i < nv; i++)
      while (__atomic_load_n(&got[i], __ATOMIC_ACQUIRE) == -2) std::this_thread::yield();
    const double ta = *std::max_element(lat.begin(), lat.end());
    if (timed) {
      a.total.v.push_back(ta);
      a.vote.v.insert(a.vote.v.end(), lat.begin(), lat.end());
      a.launches += hs_kernel_launches(ctx) - l0;
      for (int i = 0; i < nv; i++) a.mismatches += got[i] != want[i];
      a.mismatches += bad.load();
    }
    // (b) one synchronous hs_verify_rec128(n = 1) per vote from the same 16 threads
    go = 0;
    l0 = hs_kernel_launches(ctx);
    for (int t = 0; t < nth; t++)
      ts.emplace_back([&, t] {
        while (!go.load()) {
        }
        for (int i = t; i < nv; i += nth) {
          uint32_t bm = 0;
          got[i] = hs_verify_rec128(ctx, &recs[i], 1, HS_MODE_STRICT, &bm) == HS_OK ? (int)(bm & 1u) : -1;
          lat[i] = us_since(t0);
        }
      });
    t0 = clk::now();
    go = 1;
    for (auto &t : ts) t.join();
    if (timed) {
      b.total.v.push_back(*std::max_element(lat.begin(), lat.end()));
      b.vote.v.insert(b.vote.v.end(), lat.begin(), lat.end());
      b.launches += hs_kernel_launches(ctx) - l0;
      for (int i = 0; i < nv; i++) b.mismatches += got[i] != want[i];
    }
  }
  hs_queue_destroy(q);
  printf("\"committee_%d\": {\"votes\": %d, \"bursts\": %d, ", N, nv, bursts);
  a.emit("queue", bursts, false);
  b.emit("sync_verify_rec128_n1_16_threads", bursts, false);
  c.emit("cpu_oracle_1core_serial", bursts, true);
  printf("}%s", last ? "" : ", ");
  return a.mismatches + b.mismatches;
}
// ---- replica Block::verify: one certificate = 1 strict author signature + N - f batch-eq QC votes (messages.rs:54-76, :180-208)
struct cert {
  std::vector<hs_rec128> recs;  // [0] author over the block digest, [1..] the QC's votes over the QC digest
  std::vector<uint8_t> modes;
  std::vector<hs_vote> votes;   // the same votes in the shape of hs_verify_batch_shared_msg
  uint8_t qd[32];
  std::vector<uint32_t> want;   // oracle verdict bitmap of recs in their modes
};
struct committee_keys {
  int N = 0;
  std::vector<uint8_t> seeds, pks;
};
static committee_keys make_keys(int N, int salt) {
  committee_keys k;
  k.N = N;
  k.seeds.resize((size_t)N * 32);
  k.pks.resize((size_t)N * 32);
  for (int i = 0; i < N; i++)
    for (int j = 0; j < 32; j++) k.seeds[(size_t)i * 32 + j] = (uint8_t)(29 * i + 5 * j + salt + (i >> 8) * 3 + (i >> 16));
  hso_keygen_batch(k.seeds.data(), N, k.pks.data());
  return k;
}
static int ncpu() { return std::max(1, (int)std::thread::hardware_concurrency()); }
// Block of round r: author r % N signs the block digest, voters (i * 7 + r) % N sign the QC digest; 1 % of the records corrupted.
static void make_cert(const committee_keys &k, int r, cert &c) {
  const int N = k.N, f = (N - 1) / 3, nv = N - f, n = nv + 1;
  uint8_t pre[40], bd[32];
  for (int j = 0; j < 32; j++) pre[j] = (uint8_t)(r * 17 + j * 3 + 1);
  const uint64_t round = 5000 + (uint64_t)r;
  memcpy(pre + 32, &round, 8);
  hso_digest32(pre, 40, c.qd);  // Vote / QC digest = SHA-512(block hash || round)
  pre[0] ^= 0x55;
  hso_digest32(pre, 40, bd);    // stands for Block::digest
  std::vector<uint32_t> key(n);
  std::vector<uint8_t> msgs((size_t)n * 32);
  std::vector<uint64_t> off(n + 1);
  for (int i = 0; i < n; i++) {
    key[i] = (uint32_t)(i == 0 ? r % N : ((i - 1) * 7 + r) % N);
    memcpy(&msgs[(size_t)i * 32], i == 0 ? bd : c.qd, 32);
    off[i] = (uint64_t)i * 32;
  }
  off[n] = (uint64_t)n * 32;
  std::vector<uint8_t> sigs((size_t)n * 64);
  hso_sign_batch(k.seeds.data(), k.pks.data(), key.data(), msgs.data(), off.data(), n, ncpu(), sigs.data());
  c.recs.resize(n);
  c.modes.assign(n, (uint8_t)HS_MODE_BATCH_EQ);
  c.modes[0] = (uint8_t)HS_MODE_STRICT;
  c.votes.resize(nv);
  for (int i = 0; i < n; i++) {
    memcpy(c.recs[i].sig, &sigs[(size_t)i * 64], 64);
    memcpy(c.recs[i].pk, &k.pks[(size_t)key[i] * 32], 32);
    memcpy(c.recs[i].msg, &msgs[(size_t)i * 32], 32);
    if ((i * 37 + r * 11) % 100 == 0) c.recs[i].sig[(i + r) % 64] ^= 0x10;  // 1 % corrupted
    if (i) {
      memcpy(c.votes[i - 1].pk, c.recs[i].pk, 32);
      memcpy(c.votes[i - 1].sig, c.recs[i].sig, 64);
    }
  }
  std::vector<uint32_t> s((n + 31) / 32), e((n + 31) / 32);
  hso_verify_rec128_batch((const uint8_t *)c.recs.data(), n, 0, ncpu(), s.data());
  hso_verify_rec128_batch((const uint8_t *)c.recs.data(), n, 1, ncpu(), e.data());
  c.want.assign((n + 31) / 32, 0);
  for (int i = 0; i < n; i++)
    if ((((c.modes[i] ? e : s)[i >> 5]) >> (i & 31)) & 1u) c.want[i >> 5] |= 1u << (i & 31);
}
static bool bit(const std::vector<uint32_t> &b, int i) { return (b[i >> 5] >> (i & 31)) & 1u; }
// the queue's counters since `since` (hs_queue_stats), as a JSON object
static void emit_stats(hs_queue *q, const uint64_t (&since)[HS_QUEUE_STATS]) {
  static const char *names[HS_QUEUE_STATS] = {"small_launches", "small_records", "bulk_launches", "bulk_records", "slow_requests", "slow_records"};
  uint64_t s[HS_QUEUE_STATS] = {};
  hs_queue_stats(q, s);
  printf("\"queue_stats\": {");
  for (int i = 0; i < HS_QUEUE_STATS; i++) printf("\"%s\": %llu%s", names[i], (unsigned long long)(s[i] - since[i]), i + 1 < HS_QUEUE_STATS ? ", " : "");
  printf("}");
}
// The synchronous calls the shim makes for one Block today: a strict author verify + one verify_batch over the QC's votes.
static int sync_block(hs_ctx *ctx, const cert &c, std::vector<uint32_t> &bits) {
  const size_t nv = c.votes.size();
  std::vector<uint32_t> vb((nv + 31) / 32);
  uint32_t a = 0;
  int all_ok = 0;
  if (hs_verify_rec128(ctx, &c.recs[0], 1, HS_MODE_STRICT, &a) != HS_OK) return 1;
  if (hs_verify_batch_shared_msg(ctx, c.qd, c.votes.data(), nv, &all_ok, vb.data()) != HS_OK) return 1;
  bits.assign((nv + 1 + 31) / 32, 0);
  bits[0] = a & 1u;
  for (size_t i = 0; i < nv; i++)
    if (bit(vb, (int)i)) bits[(i + 1) >> 5] |= 1u << ((i + 1) & 31);
  return 0;
}
static int count_mismatch(const cert &c, const std::vector<uint32_t> &bits) {
  int m = 0;
  for (size_t i = 0; i < c.recs.size(); i++) m += bit(bits, (int)i) != bit(c.want, (int)i);
  return m;
}
static int replica_block(hs_ctx *ctx, hs_queue *q, int N, int blocks, bool last) {
  const committee_keys k = make_keys(N, 11);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  series qa, sb, cc;
  uint64_t launches = 0, s0[HS_QUEUE_STATS] = {};
  int mism_a = 0, mism_b = 0, bad = 0;
  cert c;
  hs_queue_stats(q, s0);
  for (int r = 0; r < blocks + 3; r++) {
    const bool timed = r >= 3;
    make_cert(k, r, c);
    const int n = (int)c.recs.size();
    std::vector<uint32_t> bits((n + 31) / 32);
    // (a) one hs_queue_submit_group, consumed by hs_queue_wait
    uint64_t l0 = hs_kernel_launches(ctx);
    auto t0 = clk::now();
    size_t ticket = 0;
    if (hs_queue_submit_group(q, c.recs.data(), n, c.modes.data(), nullptr, nullptr, &ticket) != HS_OK || hs_queue_wait(q, ticket, bits.data()) != HS_OK) bad++;
    const double ta = us_since(t0);
    if (timed) {
      qa.v.push_back(ta);
      launches += hs_kernel_launches(ctx) - l0;
      mism_a += count_mismatch(c, bits);
    }
    // (b) the synchronous calls
    t0 = clk::now();
    bad += sync_block(ctx, c, bits);
    const double tb = us_since(t0);
    if (timed) {
      sb.v.push_back(tb);
      mism_b += count_mismatch(c, bits);
    }
    // (c) the CPU oracle on one core: strict author verify + verify_batch of the votes
    std::vector<uint32_t> vb((n - 1 + 31) / 32);
    t0 = clk::now();
    const int au = hso_verify_strict(c.recs[0].sig, c.recs[0].pk, c.recs[0].msg, 32);
    hso_verify_batch_shared_msg(c.qd, (const uint8_t *)c.votes.data(), n - 1, 1, vb.data());
    if (timed) cc.v.push_back(us_since(t0));
    bad += au != (int)bit(c.want, 0);
  }
  const int nv = N - (N - 1) / 3;
  printf("\"committee_%d\": {\"records\": %d, \"blocks\": %d, \"queue_submit_group\": {\"p50_us\": %.1f, \"p99_us\": %.1f, \"launches_per_block\": %.2f, "
         "\"mismatches\": %d}, \"sync_strict_author_plus_verify_batch_shared_msg\": {\"p50_us\": %.1f, \"p99_us\": %.1f, \"mismatches\": %d}, "
         "\"cpu_oracle_1core\": {\"p50_us\": %.1f, \"p99_us\": %.1f}, \"errors\": %d, ",
         N, nv + 1, blocks, qa.pct(0.5), qa.pct(0.99), (double)launches / blocks, mism_a, sb.pct(0.5), sb.pct(0.99), mism_b, cc.pct(0.5), cc.pct(0.99), bad);
  emit_stats(q, s0);  // warm-up blocks included
  printf("}%s", last ? "" : ", ");
  return mism_a + mism_b + bad;
}

// ---- a Block certificate submitted in the middle of the leader's vote burst (N = 1,000: 667 votes + a 668-record Block;
// N = 10,000: 6,667 votes + a 6,668-record Block, on a ring of `ring` records)
struct blk_done {
  clk::time_point t0;
  double lat;
  std::vector<uint32_t> bits;
  std::atomic<int> done{0};
};
static void on_block(void *user, size_t, int status, const uint32_t *bitmap) {
  blk_done *b = (blk_done *)user;
  b->lat = us_since(b->t0);
  if (status == HS_OK) memcpy(b->bits.data(), bitmap, 4 * b->bits.size());
  else std::fill(b->bits.begin(), b->bits.end(), 0u);
  b->done.store(status == HS_OK ? 1 : -1, std::memory_order_release);
}
static int block_during_burst(hs_ctx *ctx, int N, size_t ring, int bursts, bool last) {
  const int f = (N - 1) / 3, nv = N - f, nth = 16;
  const committee_keys k = make_keys(N, 23);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, ring, &q) != HS_OK) return 1;
  burst_arm arm[2];
  series blk[2];
  int blk_bad[2] = {0, 0};
  std::vector<hs_rec128> votes(nv);
  std::vector<int> want(nv), got(nv);
  std::vector<double> lat(nv);
  std::vector<burst_vote> bv(nv);
  cert c;
  for (int r = 0; r < bursts + 3; r++) {
    const bool timed = r >= 3;
    make_cert(k, 1000 + r, c);  // the replica's Block (another round's certificate)
    uint8_t pre[40], d[32];
    for (int j = 0; j < 32; j++) pre[j] = (uint8_t)(r * 13 + j);
    const uint64_t round = 1000 + (uint64_t)r;
    memcpy(pre + 32, &round, 8);
    hso_digest32(pre, 40, d);
    for (int i = 0; i < nv; i++) {
      const int kk = (i * 7 + r) % N;
      hso_sign(&k.seeds[(size_t)kk * 32], d, 32, votes[i].sig);
      memcpy(votes[i].pk, &k.pks[(size_t)kk * 32], 32);
      memcpy(votes[i].msg, d, 32);
      if ((i * 37 + r * 11) % 100 == 0) votes[i].sig[(i + r) % 64] ^= 0x10;
    }
    std::vector<uint32_t> wb((nv + 31) / 32);
    hso_verify_rec128_batch((const uint8_t *)votes.data(), nv, 0, ncpu(), wb.data());
    for (int i = 0; i < nv; i++) want[i] = bit(wb, i);
    for (int a = 0; a < 2; a++) {  // a = 0: the Block through the queue; a = 1: the Block as synchronous calls
      std::atomic<int> go{0}, submitted{0}, bad{0};
      blk_done bd;
      bd.bits.assign((c.recs.size() + 31) / 32, 0);
      std::vector<std::thread> ts;
      std::fill(got.begin(), got.end(), -2);
      clk::time_point t0;
      const uint64_t l0 = hs_kernel_launches(ctx);
      for (int t = 0; t < nth; t++)
        ts.emplace_back([&, t] {
          while (!go.load()) {
          }
          for (int i = t; i < nv; i += nth) {
            bv[i] = burst_vote{t0, &lat[i], &got[i]};
            int rc;
            while ((rc = hs_queue_submit(q, &votes[i], 1, HS_MODE_STRICT, on_vote, &bv[i], nullptr)) == HS_ERR_NOMEM) std::this_thread::yield();
            if (rc != HS_OK) bad++;
            submitted++;
          }
        });
      ts.emplace_back([&] {  // the replica's connection task: its Block arrives when half the votes are in
        while (submitted.load() < nv / 2) {
        }
        bd.t0 = clk::now();
        if (a == 0) {
          if (hs_queue_submit_group(q, c.recs.data(), c.recs.size(), c.modes.data(), on_block, &bd, nullptr) != HS_OK) bd.done.store(-1);
        } else {
          std::vector<uint32_t> bits;
          const int rc = sync_block(ctx, c, bits);
          bd.lat = us_since(bd.t0);
          if (rc == 0) bd.bits = bits;
          bd.done.store(rc == 0 ? 1 : -1);
        }
      });
      t0 = clk::now();
      go = 1;
      for (auto &t : ts) t.join();
      for (int i = 0; i < nv; i++)
        while (__atomic_load_n(&got[i], __ATOMIC_ACQUIRE) == -2) std::this_thread::yield();
      while (bd.done.load(std::memory_order_acquire) == 0) std::this_thread::yield();
      if (timed) {
        arm[a].total.v.push_back(*std::max_element(lat.begin(), lat.end()));
        arm[a].vote.v.insert(arm[a].vote.v.end(), lat.begin(), lat.end());
        arm[a].launches += hs_kernel_launches(ctx) - l0;
        for (int i = 0; i < nv; i++) arm[a].mismatches += got[i] != want[i];
        arm[a].mismatches += bad.load();
        blk[a].v.push_back(bd.lat);
        blk_bad[a] += (bd.done.load() != 1) + count_mismatch(c, bd.bits);
      }
    }
  }
  printf("\"committee_%d\": {\"ring_records\": %zu, \"votes\": %d, \"block_records\": %zu, \"bursts\": %d, ", N, ring, nv, c.recs.size(), bursts);
  const char *names[2] = {"block_via_queue_submit_group", "block_via_synchronous_calls_other_thread"};
  for (int a = 0; a < 2; a++) {
    printf("\"%s\": {\"block_p50_us\": %.1f, \"block_p99_us\": %.1f, \"block_mismatches\": %d, ", names[a], blk[a].pct(0.5), blk[a].pct(0.99), blk_bad[a]);
    arm[a].emit("votes", bursts, true);
    printf("}, ");
  }
  const uint64_t zero[HS_QUEUE_STATS] = {};
  emit_stats(q, zero);  // both arms' votes and the queued blocks, warm-up bursts included
  printf("}%s", last ? "" : ", ");
  hs_queue_destroy(q);
  return arm[0].mismatches + arm[1].mismatches + blk_bad[0] + blk_bad[1];
}
// ---- certificate preimages: a TC (N - f strict votes, each over its own 16-byte preimage tc.round || high_qc_round) and a Block
// with a TC (strict author over the Block preimage, N - f batch-eq QC votes over one 40-byte preimage, N - f strict TC votes), 1 %
// of the signatures corrupted.  Three arms per certificate, timed from the start of the caller's work to the verdict:
//   (a) the caller hashes every distinct preimage on its own thread (hso_digest32: the oracle's C restatement of SHA-512, not the
//       reference's sha2 crate), packs hs_rec128 records and calls hs_queue_submit_group + hs_queue_wait (the queue path until now);
//   (b) hs_queue_submit_msgs with the preimages + hs_queue_wait (the Digests are computed by k_queue_digests);
//   (c) the synchronous hs_verify_tcs (TC) / hs_verify_groups (Block).
// CPU time of the caller's thread per certificate: CLOCK_THREAD_CPUTIME_ID over a back-to-back pass of 400 certificates per arm.
struct pre_cert {
  std::vector<uint8_t> pre, sig, pk, modes;
  std::vector<uint64_t> off, hq;  // hq: high_qc_round per TC vote (the TC shape only)
  std::vector<uint32_t> midx, want;
  uint64_t tc_round = 0;
};
static double thread_cpu_us() {
  timespec ts;
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &ts);
  return ts.tv_sec * 1e6 + ts.tv_nsec / 1e3;
}
static void make_pre_cert(const committee_keys &k, int r, bool block, pre_cert &c) {
  const int N = k.N, nv = N - (N - 1) / 3;
  c = pre_cert{};
  c.tc_round = 7000 + (uint64_t)r;
  auto add_pre = [&](const uint8_t *p, size_t len) {
    c.pre.insert(c.pre.end(), p, p + len);
    c.off.push_back(c.pre.size());
  };
  c.off.push_back(0);
  std::vector<uint32_t> key;
  if (block) {
    uint8_t bp[32 + 8 + 64 + 32], qp[40];  // Block::digest preimage (author, round, payload digests, qc hash), QC digest preimage
    for (size_t j = 0; j < sizeof(bp); j++) bp[j] = (uint8_t)(r * 5 + j * 11 + 3);
    for (size_t j = 0; j < sizeof(qp); j++) qp[j] = (uint8_t)(r * 7 + j * 13 + 1);
    add_pre(bp, sizeof(bp));
    add_pre(qp, sizeof(qp));
    key.push_back((uint32_t)(r % N));
    c.midx.push_back(0);
    c.modes.push_back(HS_MODE_STRICT);
    for (int i = 0; i < nv; i++) {
      key.push_back((uint32_t)((i * 7 + r) % N));
      c.midx.push_back(1);
      c.modes.push_back(HS_MODE_BATCH_EQ);
    }
  }
  for (int i = 0; i < nv; i++) {  // the TC's votes
    const uint64_t hq = c.tc_round - 1 - (uint64_t)((i * 3 + r) % 5);
    uint8_t tp[16];
    memcpy(tp, &c.tc_round, 8);
    memcpy(tp + 8, &hq, 8);
    add_pre(tp, 16);
    c.hq.push_back(hq);
    key.push_back((uint32_t)((i * 5 + r + 1) % N));
    c.midx.push_back((uint32_t)(c.off.size() - 2));
    c.modes.push_back(HS_MODE_STRICT);
  }
  const size_t n = key.size(), n_msgs = c.off.size() - 1;
  std::vector<uint8_t> dig(n_msgs * 32), msgs(n * 32);
  for (size_t j = 0; j < n_msgs; j++) hso_digest32(&c.pre[c.off[j]], c.off[j + 1] - c.off[j], &dig[j * 32]);
  std::vector<uint64_t> moff(n + 1);
  for (size_t i = 0; i <= n; i++) moff[i] = 32 * i;
  for (size_t i = 0; i < n; i++) memcpy(&msgs[i * 32], &dig[c.midx[i] * 32], 32);
  c.sig.resize(n * 64);
  c.pk.resize(n * 32);
  hso_sign_batch(k.seeds.data(), k.pks.data(), key.data(), msgs.data(), moff.data(), n, ncpu(), c.sig.data());
  std::vector<uint8_t> recs(n * 128);
  for (size_t i = 0; i < n; i++) {
    if ((i * 37 + r * 11) % 100 == 0) c.sig[i * 64 + (i + r) % 64] ^= 0x10;  // 1 % corrupted
    memcpy(&c.pk[i * 32], &k.pks[(size_t)key[i] * 32], 32);
    memcpy(&recs[i * 128], &c.sig[i * 64], 64);
    memcpy(&recs[i * 128 + 64], &c.pk[i * 32], 32);
    memcpy(&recs[i * 128 + 96], &msgs[i * 32], 32);
  }
  std::vector<uint32_t> s((n + 31) / 32), e((n + 31) / 32);
  hso_verify_rec128_batch(recs.data(), n, 0, ncpu(), s.data());
  hso_verify_rec128_batch(recs.data(), n, 1, ncpu(), e.data());
  c.want.assign((n + 31) / 32, 0);
  for (size_t i = 0; i < n; i++)
    if ((((c.modes[i] ? e : s)[i >> 5]) >> (i & 31)) & 1u) c.want[i >> 5] |= 1u << (i & 31);
}
static int certificate_preimages(hs_ctx *ctx, hs_queue *q, int N, bool block, int certs, int cpu_reps, bool last) {
  const committee_keys k = make_keys(N, 31);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  series lat[3], cpu[3];
  int mism[3] = {0, 0, 0}, bad = 0;
  uint64_t s0[HS_QUEUE_STATS] = {}, d0[HS_QUEUE_DIGEST_STATS] = {}, d1[HS_QUEUE_DIGEST_STATS] = {};
  hs_queue_stats(q, s0);
  hs_queue_digest_stats(q, d0);
  pre_cert c;
  std::vector<hs_rec128> recs;
  std::vector<uint8_t> dig;
  for (int r = 0; r < certs + 3; r++) {
    const bool timed = r >= 3;
    make_pre_cert(k, r, block, c);
    const size_t n = c.midx.size(), n_msgs = c.off.size() - 1;
    std::vector<uint32_t> bits((n + 31) / 32);
    // one arm on certificate c; with `timed`, its latency and mismatches are recorded
    auto run_arm = [&](int a, bool timed) {
      std::fill(bits.begin(), bits.end(), 0u);
      const auto t0 = clk::now();
      int rc = HS_OK;
      size_t ticket = 0;
      if (a == 0) {  // (a) hash on the caller's thread, pack records, submit_group
        dig.resize(n_msgs * 32);
        for (size_t j = 0; j < n_msgs; j++) hso_digest32(&c.pre[c.off[j]], c.off[j + 1] - c.off[j], &dig[j * 32]);
        recs.resize(n);
        for (size_t i = 0; i < n; i++) {
          memcpy(recs[i].sig, &c.sig[i * 64], 64);
          memcpy(recs[i].pk, &c.pk[i * 32], 32);
          memcpy(recs[i].msg, &dig[c.midx[i] * 32], 32);
        }
        rc = hs_queue_submit_group(q, recs.data(), n, c.modes.data(), nullptr, nullptr, &ticket);
        if (rc == HS_OK) rc = hs_queue_wait(q, ticket, bits.data());
      } else if (a == 1) {  // (b) the preimages, hashed on the GPU
        rc = hs_queue_submit_msgs(q, c.pre.data(), c.off.data(), n_msgs, c.sig.data(), c.pk.data(), c.midx.data(), c.modes.data(), n, nullptr, nullptr,
                                  &ticket);
        if (rc == HS_OK) rc = hs_queue_wait(q, ticket, bits.data());
      } else if (!block) {  // (c) synchronous: one TC
        uint32_t tcb = 0;
        rc = hs_verify_tcs(ctx, &c.tc_round, 1, c.pk.data(), nullptr, c.sig.data(), c.hq.data(), std::vector<uint32_t>(n, 0).data(), n, bits.data(), &tcb);
      } else {  // (c) synchronous: one Block with its QC and TC
        uint32_t gb = 0;
        rc = hs_verify_groups(ctx, c.pre.data(), c.off.data(), n_msgs, c.sig.data(), c.pk.data(), nullptr, c.midx.data(), std::vector<uint32_t>(n, 0).data(),
                              c.modes.data(), n, 1, bits.data(), &gb);
      }
      const double t = us_since(t0);
      bad += rc != HS_OK;
      if (timed) {
        lat[a].v.push_back(t);
        for (size_t i = 0; i < n; i++) mism[a] += bit(bits, (int)i) != bit(c.want, (int)i);
      }
    };
    for (int a = 0; a < 3; a++) run_arm(a, timed);
    if (r == certs + 2) {  // the caller thread's CPU time: a back-to-back pass per arm (the thread CPU clock may tick coarsely)
      for (int a = 0; a < 3; a++) {
        const double c0 = thread_cpu_us();
        for (int rep = 0; rep < cpu_reps; rep++) run_arm(a, false);
        cpu[a].v.push_back((thread_cpu_us() - c0) / cpu_reps);
      }
    }
  }
  hs_queue_digest_stats(q, d1);
  const int nv = N - (N - 1) / 3;
  printf("\"%s_committee_%d\": {\"records\": %d, \"preimages\": %d, \"certificates\": %d, \"cpu_pass_certificates\": %d, ", block ? "block_with_tc" : "tc", N,
         block ? 1 + 2 * nv : nv, block ? 2 + nv : nv, certs, cpu_reps);
  const char *names[3] = {"a_caller_hashes_then_submit_group", "b_submit_msgs", block ? "c_sync_verify_groups" : "c_sync_verify_tcs"};
  for (int a = 0; a < 3; a++)
    printf("\"%s\": {\"p50_us\": %.1f, \"p99_us\": %.1f, \"caller_cpu_us_per_cert\": %.1f, \"mismatches\": %d}, ", names[a], lat[a].pct(0.5), lat[a].pct(0.99),
           cpu[a].mean(), mism[a]);
  printf("\"errors\": %d, \"digest_stats\": {\"digest_launches\": %llu, \"preimages\": %llu, \"preimage_bytes\": %llu, \"msgs_requests\": %llu}, ", bad,
         (unsigned long long)(d1[0] - d0[0]), (unsigned long long)(d1[1] - d0[1]), (unsigned long long)(d1[2] - d0[2]), (unsigned long long)(d1[3] - d0[3]));
  emit_stats(q, s0);  // warm-up certificates included
  printf("}%s", last ? "" : ", ");
  return mism[0] + mism[1] + mism[2] + bad;
}

static std::string gpu_identity() {  // name and enforced power limit, read in the same run
  std::string s;
  if (FILE *p = popen("nvidia-smi --query-gpu=name,power.limit --format=csv,noheader -i 0 2>/dev/null", "r")) {
    char buf[256];
    while (fgets(buf, sizeof(buf), p)) s += buf;
    pclose(p);
  }
  while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back();
  for (char &ch : s)
    if (ch == '"') ch = '\'';
  return s.empty() ? "unknown" : s;
}

// The certificate_preimages section alone (argv[3] == "certificate_preimages"), or after the others.
static int run_certificate_preimages(hs_ctx *ctx, int certs) {
  timespec res;
  clock_getres(CLOCK_THREAD_CPUTIME_ID, &res);
  printf("\"certificate_preimages\": {\"gpu\": \"%s\", \"ring_records\": 16384, \"caller_sha512\": \"oracle C restatement (hso_digest32), not the sha2 crate\", "
         "\"thread_cpu_clock_res_ns\": %ld, ",
         gpu_identity().c_str(), (long)(res.tv_sec * 1000000000L + res.tv_nsec));
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 16384, &q) != HS_OK) return 1;
  int bad = 0;
  for (int block = 0; block < 2; block++)
    for (int N : {4, 100, 250, 500, 750}) bad += certificate_preimages(ctx, q, N, block == 1, certs, 400, block == 1 && N == 750);
  hs_queue_destroy(q);
  printf("}");
  return bad;
}

// ---- view change: every validator's Timeout at once, nearly all carrying the same high_qc (consensus/src/core.rs local_timeout
// -> handle_timeout).  One burst = N Timeout frames released together to 16 threads (one per connection task): record 0 the author's
// strict signature over round || high_qc.round (16 bytes), records 1.. the high_qc's N - f batch-eq votes over hash || round (40
// bytes).  1 % of the author signatures are corrupted.  Each burst has a new QC: cold = first seen in the burst; warm = the Block
// carrying it went through the queue first, and a tenth of the Timeouts carry a copy of the QC with one bad vote (each must be
// rejected, and that QC must never enter the cache).  Arms:
//   (a) the queue without the cache, as the Rust module does today: a Timeout of more than GROUP_MAX_SIGS = 502 records, or one the
//       queue refuses, is verified synchronously (a strict author verify + hs_verify_batch_shared_msg);
//   (b) the queue with the certificate cache (hs_queue_submit_msgs, the same synchronous fallback on a refusal);
//   (c) the synchronous batched calls of Core::verify_timeouts: one hs_verify_tcs for every author + one QC verify per distinct QC.
// Burst time = release -> the last Timeout's verdict.  Signatures verified = the records the queue's launches and slow path carried
// plus the synchronous ones.
#define VC_THREADS 16
#define VC_GROUP_MAX_SIGS 502
struct vc_qc {
  uint8_t pre[40], dig[32];
  std::vector<uint8_t> sig, pk;  // nv x 64, nv x 32
  std::vector<hs_vote> votes;
  std::vector<uint32_t> want;    // oracle, batch-eq
};
struct vc_burst {
  int N = 0, nv = 0;
  uint64_t round = 0, hq = 0;
  std::vector<uint8_t> a_sig, a_pk;  // N authors
  std::vector<uint32_t> a_want;      // oracle, strict
  vc_qc qc[2];                       // [1]: [0] with one bad vote
  std::vector<uint8_t> bad;          // Timeout i carries qc[1]
};
static void vc_make(const committee_keys &k, int b, bool bad_qc, vc_burst &v) {
  const int N = k.N, nv = N - (N - 1) / 3;
  v.N = N;
  v.nv = nv;
  v.round = 90000 + (uint64_t)b * 3 + (bad_qc ? 1 : 0);
  v.hq = v.round - 1;
  uint8_t tp[16];
  memcpy(tp, &v.round, 8);
  memcpy(tp + 8, &v.hq, 8);
  uint8_t td[32];
  hso_digest32(tp, 16, td);
  std::vector<uint32_t> key(N);
  std::vector<uint8_t> msgs((size_t)N * 32);
  std::vector<uint64_t> off(N + 1);
  for (int i = 0; i < N; i++) {
    key[i] = (uint32_t)i;
    memcpy(&msgs[(size_t)i * 32], td, 32);
  }
  for (int i = 0; i <= N; i++) off[i] = (uint64_t)i * 32;
  v.a_sig.resize((size_t)N * 64);
  v.a_pk.assign(k.pks.begin(), k.pks.end());
  hso_sign_batch(k.seeds.data(), k.pks.data(), key.data(), msgs.data(), off.data(), N, ncpu(), v.a_sig.data());
  for (int i = 0; i < N; i++)
    if ((i * 37 + b * 11) % 100 == 0) v.a_sig[(size_t)i * 64 + (i + b) % 64] ^= 0x10;  // 1 % of the authors corrupted
  std::vector<uint8_t> recs((size_t)N * 128);
  for (int i = 0; i < N; i++) {
    memcpy(&recs[(size_t)i * 128], &v.a_sig[(size_t)i * 64], 64);
    memcpy(&recs[(size_t)i * 128 + 64], &v.a_pk[(size_t)i * 32], 32);
    memcpy(&recs[(size_t)i * 128 + 96], td, 32);
  }
  v.a_want.assign((N + 31) / 32, 0);
  hso_verify_rec128_batch(recs.data(), N, 0, ncpu(), v.a_want.data());
  vc_qc &q = v.qc[0];
  for (int j = 0; j < 32; j++) q.pre[j] = (uint8_t)(b * 19 + j * 7 + (bad_qc ? 101 : 3));
  memcpy(q.pre + 32, &v.hq, 8);
  hso_digest32(q.pre, 40, q.dig);
  for (int i = 0; i < nv; i++) {
    key[i] = (uint32_t)((i * 7 + b) % N);
    memcpy(&msgs[(size_t)i * 32], q.dig, 32);
  }
  q.sig.resize((size_t)nv * 64);
  q.pk.resize((size_t)nv * 32);
  hso_sign_batch(k.seeds.data(), k.pks.data(), key.data(), msgs.data(), off.data(), nv, ncpu(), q.sig.data());
  for (int i = 0; i < nv; i++) memcpy(&q.pk[(size_t)i * 32], &k.pks[(size_t)key[i] * 32], 32);
  v.qc[1] = q;
  v.qc[1].sig[(size_t)(nv / 2) * 64 + 40] ^= 0x04;  // one bad vote
  for (vc_qc &x : v.qc) {
    x.votes.resize(nv);
    recs.resize((size_t)nv * 128);
    for (int i = 0; i < nv; i++) {
      memcpy(x.votes[i].pk, &x.pk[(size_t)i * 32], 32);
      memcpy(x.votes[i].sig, &x.sig[(size_t)i * 64], 64);
      memcpy(&recs[(size_t)i * 128], &x.sig[(size_t)i * 64], 64);
      memcpy(&recs[(size_t)i * 128 + 64], &x.pk[(size_t)i * 32], 32);
      memcpy(&recs[(size_t)i * 128 + 96], x.dig, 32);
    }
    x.want.assign((nv + 31) / 32, 0);
    hso_verify_rec128_batch(recs.data(), nv, 1, ncpu(), x.want.data());
  }
  v.bad.assign(N, 0);
  if (bad_qc)
    for (int i = 7; i < N; i += 10) v.bad[i] = 1;
}
struct vc_arm {
  series t;
  uint64_t sync_sigs = 0, fallbacks = 0;
  int mismatches = 0, bad_accepted = 0, errors = 0;
};
// The synchronous Timeout::verify of the Rust module's fallback: a strict author verify + verify_batch over the QC's votes.
static int vc_sync_timeout(hs_ctx *ctx, const vc_burst &v, int i, std::vector<uint32_t> &bits) {
  const vc_qc &q = v.qc[v.bad[i]];
  hs_rec128 a;
  memcpy(a.sig, &v.a_sig[(size_t)i * 64], 64);
  memcpy(a.pk, &v.a_pk[(size_t)i * 32], 32);
  uint8_t tp[16];
  memcpy(tp, &v.round, 8);
  memcpy(tp + 8, &v.hq, 8);
  hso_digest32(tp, 16, a.msg);
  uint32_t ab = 0;
  int ok = 0;
  std::vector<uint32_t> vb((v.nv + 31) / 32);
  if (hs_verify_rec128(ctx, &a, 1, HS_MODE_STRICT, &ab) != HS_OK) return 1;
  if (hs_verify_batch_shared_msg(ctx, q.dig, q.votes.data(), v.nv, &ok, vb.data()) != HS_OK) return 1;
  std::fill(bits.begin(), bits.end(), 0u);
  bits[0] = ab & 1u;
  for (int k = 0; k < v.nv; k++)
    if (bit(vb, k)) bits[(k + 1) >> 5] |= 1u << ((k + 1) & 31);
  return 0;
}
static void vc_check(const vc_burst &v, int i, const std::vector<uint32_t> &bits, std::atomic<int> &mism, std::atomic<int> &bad_acc) {
  const vc_qc &q = v.qc[v.bad[i]];
  int m = bit(bits, 0) != bit(v.a_want, i), all = bit(bits, 0);
  for (int k = 0; k < v.nv; k++) {
    m += bit(bits, k + 1) != bit(q.want, k);
    all &= bit(bits, k + 1);
  }
  mism += m;
  bad_acc += v.bad[i] && all;
}
// One burst through a queue (arms a and b): thread t takes Timeouts t, t + 16, ...; it submits each, then waits for each.
static double vc_queue_burst(hs_ctx *ctx, hs_queue *q, bool cache, const vc_burst &v, vc_arm &arm) {
  const int N = v.N, n = 1 + v.nv;
  std::atomic<int> go{0}, mism{0}, bad_acc{0}, errs{0};
  std::atomic<uint64_t> sync_sigs{0}, fallbacks{0};
  uint8_t pre[56];
  memcpy(pre, &v.round, 8);
  memcpy(pre + 8, &v.hq, 8);
  const uint64_t off[3] = {0, 16, 56};
  std::vector<std::thread> th;
  for (int t = 0; t < VC_THREADS; t++)
    th.emplace_back([&, t] {
      std::vector<uint8_t> sig((size_t)n * 64), pk((size_t)n * 32), modes(n, HS_MODE_BATCH_EQ), p(pre, pre + 56);
      std::vector<uint32_t> midx(n, 1), bits((n + 31) / 32);
      midx[0] = 0;
      modes[0] = HS_MODE_STRICT;
      std::vector<std::pair<int, size_t>> tickets;
      while (!go.load()) {
      }
      for (int i = t; i < N; i += VC_THREADS) {
        const vc_qc &qc = v.qc[v.bad[i]];
        int rc = HS_ERR_ARG;
        size_t ticket = 0;
        if (cache || n <= VC_GROUP_MAX_SIGS) {
          memcpy(p.data() + 16, qc.pre, 40);
          memcpy(sig.data(), &v.a_sig[(size_t)i * 64], 64);
          memcpy(pk.data(), &v.a_pk[(size_t)i * 32], 32);
          memcpy(sig.data() + 64, qc.sig.data(), qc.sig.size());
          memcpy(pk.data() + 32, qc.pk.data(), qc.pk.size());
          rc = hs_queue_submit_msgs(q, p.data(), off, 2, sig.data(), pk.data(), midx.data(), modes.data(), n, nullptr, nullptr, &ticket);
        }
        if (rc == HS_OK) {
          tickets.emplace_back(i, ticket);
          continue;
        }
        if (rc != HS_ERR_NOMEM && rc != HS_ERR_ARG) errs++;
        fallbacks += cache || n <= VC_GROUP_MAX_SIGS;
        errs += vc_sync_timeout(ctx, v, i, bits);
        sync_sigs += n;
        vc_check(v, i, bits, mism, bad_acc);
      }
      for (auto &[i, ticket] : tickets) {
        std::fill(bits.begin(), bits.end(), 0u);
        errs += hs_queue_wait(q, ticket, bits.data()) != HS_OK;
        vc_check(v, i, bits, mism, bad_acc);
      }
    });
  const auto t0 = clk::now();
  go = 1;
  for (std::thread &x : th) x.join();
  const double us = us_since(t0);
  arm.mismatches += mism;
  arm.bad_accepted += bad_acc;
  arm.errors += errs;
  arm.sync_sigs += sync_sigs;
  arm.fallbacks += fallbacks;
  return us;
}
// Arm (c): the Timeouts' authors in one hs_verify_tcs (one TC of N votes over round || high_qc.round), then each distinct QC once.
static double vc_sync_burst(hs_ctx *ctx, const vc_burst &v, vc_arm &arm) {
  const int N = v.N;
  std::vector<uint32_t> ab((N + 31) / 32), vb[2], tcidx(N, 0);
  std::vector<uint64_t> hq(N, v.hq);
  const bool two = std::count(v.bad.begin(), v.bad.end(), 1) > 0;
  const auto t0 = clk::now();
  uint32_t tcb = 0;
  arm.errors += hs_verify_tcs(ctx, &v.round, 1, v.a_pk.data(), nullptr, v.a_sig.data(), hq.data(), tcidx.data(), N, ab.data(), &tcb) != HS_OK;
  for (int k = 0; k < 1 + two; k++) {
    int ok = 0;
    vb[k].assign((v.nv + 31) / 32, 0);
    arm.errors += hs_verify_batch_shared_msg(ctx, v.qc[k].dig, v.qc[k].votes.data(), v.nv, &ok, vb[k].data()) != HS_OK;
  }
  const double us = us_since(t0);
  arm.sync_sigs += N + (uint64_t)(1 + two) * v.nv;
  std::atomic<int> mism{0}, bad_acc{0};
  std::vector<uint32_t> bits((1 + v.nv + 31) / 32);
  for (int i = 0; i < N; i++) {
    std::fill(bits.begin(), bits.end(), 0u);
    bits[0] = bit(ab, i);
    for (int k = 0; k < v.nv; k++)
      if (bit(vb[v.bad[i]], k)) bits[(k + 1) >> 5] |= 1u << ((k + 1) & 31);
    vc_check(v, i, bits, mism, bad_acc);
  }
  arm.mismatches += mism;
  arm.bad_accepted += bad_acc;
  return us;
}
static uint64_t queue_sigs(hs_queue *q) {  // records the queue's launches and slow path carried
  uint64_t s[HS_QUEUE_STATS] = {};
  hs_queue_stats(q, s);
  return s[1] + s[3] + s[5];
}
static int view_change(hs_ctx *ctx, int N, int bursts, bool warm, bool last) {
  const committee_keys k = make_keys(N, 41);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  hs_queue *qa = nullptr, *qb = nullptr;
  if (hs_queue_create(ctx, 0, &qa) != HS_OK || hs_queue_create(ctx, 0, &qb) != HS_OK) return 1;
  hs_queue_cert_cache(qb, 64u << 20);
  vc_arm arm[3];
  uint64_t qsig[2] = {0, 0}, c0[HS_QUEUE_CERT_STATS] = {}, c1[HS_QUEUE_CERT_STATS] = {};
  int bad = 0, inserted_in_bursts = 0;
  vc_burst v;
  for (int b = 0; b < bursts + 2; b++) {
    const bool timed = b >= 2;
    vc_make(k, b, warm, v);
    if (warm) {  // the Block carrying the QC, through the cached queue first (not timed)
      uint8_t bp[136 + 40];
      for (int j = 0; j < 136; j++) bp[j] = (uint8_t)(b * 3 + j);
      memcpy(bp + 136, v.qc[0].pre, 40);
      const uint64_t off[3] = {0, 136, 176};
      const int n = 1 + v.nv;
      std::vector<uint8_t> sig((size_t)n * 64), pk((size_t)n * 32), modes(n, HS_MODE_BATCH_EQ);
      std::vector<uint32_t> midx(n, 1), bits((n + 31) / 32);
      midx[0] = 0;
      modes[0] = HS_MODE_STRICT;
      memcpy(sig.data() + 64, v.qc[0].sig.data(), v.qc[0].sig.size());
      memcpy(pk.data() + 32, v.qc[0].pk.data(), v.qc[0].pk.size());
      size_t ticket = 0;
      bad += hs_queue_submit_msgs(qb, bp, off, 2, sig.data(), pk.data(), midx.data(), modes.data(), n, nullptr, nullptr, &ticket) != HS_OK;
      hs_queue_wait(qb, ticket, bits.data());
    }
    uint64_t s0[2] = {queue_sigs(qa), queue_sigs(qb)};
    uint64_t i0[HS_QUEUE_CERT_STATS] = {}, i1[HS_QUEUE_CERT_STATS] = {};
    hs_queue_cert_stats(qb, i0);
    if (timed && b == 2) memcpy(c0, i0, sizeof(c0));
    vc_arm scratch[3];
    vc_arm *use = timed ? arm : scratch;
    const double ta = vc_queue_burst(ctx, qa, false, v, use[0]);
    const double tb = vc_queue_burst(ctx, qb, true, v, use[1]);
    const double tc = vc_sync_burst(ctx, v, use[2]);
    hs_queue_cert_stats(qb, i1);
    if (timed) {
      arm[0].t.v.push_back(ta);
      arm[1].t.v.push_back(tb);
      arm[2].t.v.push_back(tc);
      qsig[0] += queue_sigs(qa) - s0[0];
      qsig[1] += queue_sigs(qb) - s0[1];
      inserted_in_bursts += (int)(i1[4] - i0[4]);
    }
    for (vc_arm &a : scratch) bad += a.mismatches + a.bad_accepted + a.errors;
  }
  hs_queue_cert_stats(qb, c1);
  const int f = (N - 1) / 3;
  printf("\"%s_committee_%d\": {\"timeouts_per_burst\": %d, \"records_per_timeout\": %d, \"bad_qc_timeouts_per_burst\": %d, \"bursts\": %d, ", warm ? "warm" : "cold", N, N,
         1 + N - f, warm ? (N + 2) / 10 : 0, bursts);
  const char *names[3] = {"a_queue_no_cache_sync_fallback", "b_queue_cert_cache", "c_sync_verify_tcs_plus_qc"};
  for (int a = 0; a < 3; a++) {
    const uint64_t sigs = (a < 2 ? qsig[a] : 0) + arm[a].sync_sigs;
    printf("\"%s\": {\"burst_p50_us\": %.1f, \"burst_p99_us\": %.1f, \"signatures_verified_per_burst\": %.0f, \"sync_fallbacks_per_burst\": %.1f, "
           "\"mismatches\": %d, \"bad_qc_timeouts_accepted\": %d, \"errors\": %d}, ",
           names[a], arm[a].t.pct(0.5), arm[a].t.pct(0.99), (double)sigs / bursts, (double)arm[a].fallbacks / bursts, arm[a].mismatches, arm[a].bad_accepted,
           arm[a].errors);
    bad += arm[a].mismatches + arm[a].bad_accepted + arm[a].errors;
  }
  static const char *cn[HS_QUEUE_CERT_STATS] = {"lookups", "hits", "joins", "records_answered", "inserted", "bytes_held"};
  printf("\"cert_stats\": {");
  for (int i = 0; i < HS_QUEUE_CERT_STATS; i++)
    printf("\"%s\": %llu%s", cn[i], (unsigned long long)(i == 5 ? c1[i] : c1[i] - c0[i]), i + 1 < HS_QUEUE_CERT_STATS ? ", " : "");
  printf("}, \"inserted_during_bursts\": %d}%s", inserted_in_bursts, last ? "" : ", ");
  // every burst has a new QC: cold inserts it once per burst, warm inserted it before the burst and never inserts the bad copy
  bad += inserted_in_bursts != (warm ? 0 : bursts);
  hs_queue_destroy(qa);
  hs_queue_destroy(qb);
  return bad;
}
static int run_view_change(hs_ctx *ctx, int bursts) {
  printf("\"view_change\": {\"gpu\": \"%s\", \"threads\": %d, \"ring_records\": 4096, \"cache_bytes\": %u, ", gpu_identity().c_str(), VC_THREADS, 64u << 20);
  int bad = 0;
  for (int warm = 0; warm < 2; warm++)
    for (int N : {100, 1000, 4000}) bad += view_change(ctx, N, N == 100 ? 2 * bursts : bursts, warm == 1, warm == 1 && N == 4000);
  printf("}");
  return bad;
}

// The queue's signature-cache counters since `since` (hs_queue_sig_stats), as a JSON object.
static void emit_sig_stats(hs_queue *q, const uint64_t (&since)[HS_QUEUE_SIG_STATS], const char *key = "sig_stats") {
  static const char *names[HS_QUEUE_SIG_STATS] = {"probed", "hits", "inserts", "evictions", "entries_held"};
  uint64_t s[HS_QUEUE_SIG_STATS] = {};
  hs_queue_sig_stats(q, s);
  printf("\"%s\": {", key);
  for (int i = 0; i < HS_QUEUE_SIG_STATS; i++)
    printf("\"%s\": %llu%s", names[i], (unsigned long long)(i == 4 ? s[i] : s[i] - since[i]), i + 1 < HS_QUEUE_SIG_STATS ? ", " : "");
  printf("}");
}

// ---- the cost of a probe that misses (alone with argv[3] = sig_cache_cost): the leader vote burst (N = 100, 1,000) and
// replica_block (N = 100 .. 6,000) with the signature cache off, then on.  Every section gets a queue of its own (the committees
// share keys, so one queue would see the same votes again), and within one every vote and every Block is new: every probe misses
// and every accepted record is inserted, so the difference is what the probe and the insert cost.
#define SIG_COST_ENTRIES (1u << 16)
static int run_sig_cache_cost(hs_ctx *ctx, int bursts) {
  printf("\"sig_cache_cost\": {\"gpu\": \"%s\", \"entries\": %u, ", gpu_identity().c_str(), SIG_COST_ENTRIES);
  int bad = 0;
  for (int on = 0; on < 2; on++) {
    g_sig_entries = on ? SIG_COST_ENTRIES : 0;
    printf("\"%s\": {\"leader_vote_burst\": {", on ? "cache_on" : "cache_off");
    for (int N : {100, 1000}) bad += vote_burst(ctx, N, bursts, N == 1000);
    printf("}, \"replica_block\": {\"ring_records\": 16384, ");
    for (int N : {100, 1000, 3000, 6000}) {
      hs_queue *q = nullptr;
      if (hs_queue_create(ctx, 16384, &q) != HS_OK || (on && hs_queue_sig_cache(q, SIG_COST_ENTRIES) != HS_OK)) return bad + 1;
      const uint64_t z[HS_QUEUE_SIG_STATS] = {};
      bad += replica_block(ctx, q, N, bursts, false);
      const std::string key = "sig_stats_committee_" + std::to_string(N);
      emit_sig_stats(q, z, key.c_str());
      printf("%s", N == 6000 ? "" : ", ");
      hs_queue_destroy(q);
    }
    printf("}}%s", on ? "" : ", ");
  }
  g_sig_entries = 0;
  printf("}");
  return bad;
}

// ---- TC after Timeouts (alone with argv[3] = tc_after_timeouts): one view change per round at N = 100, 1,000 and 4,000.  N
// Timeouts go through the queue first (16 threads, hs_queue_submit_msgs, certificate cache on): record 0 the author's strict
// signature over round || high_qc.round (16 bytes), records 1.. the shared high_qc's N - f batch-eq votes over hash || round (40
// bytes); 1 % of the author signatures are corrupted.  Then the TC: the first N - f Timeouts' (author, signature, high_qc.round)
// triples, strict, each over its own 16-byte preimage (the corrupted ones included: they must be rejected again).  Then the Block
// carrying that TC: a strict author signature over the Block preimage, the QC's votes batch-eq, the TC's votes strict.  The TC and
// the Block are timed (submit -> verdict, one at a time) in three arms:
//   (a) synchronous: hs_verify_tcs (TC) / hs_verify_groups (Block), no Timeouts needed;
//   (b) the queue without the signature cache;  (c) the queue with it.
// Each of (b) and (c) has its own queue (16,384 records, certificate cache 64 MB) that saw the round's Timeouts first.
struct tc_round {
  std::vector<uint8_t> qsig, qpk, asig, apk, qp, bp, bsig;  // QC votes, Timeout authors (N), QC preimage, Block preimage, Block author
  std::vector<uint8_t> tpre;                                // the Timeouts' 16-byte preimages (all equal: one high_qc)
  std::vector<uint32_t> a_want, q_want;                     // oracle: authors strict, QC votes batch-eq
  uint64_t round = 0, hq = 0;
  uint32_t bkey = 0;
  bool b_want = false;
};
static void tc_make(const committee_keys &k, int r, tc_round &t) {
  const int N = k.N, nv = N - (N - 1) / 3;
  t.round = 9000 + (uint64_t)r * 2;
  t.hq = t.round - 1;
  t.qp.resize(40);
  for (int j = 0; j < 32; j++) t.qp[j] = (uint8_t)(r * 19 + j * 5 + 2);
  memcpy(&t.qp[32], &t.hq, 8);
  t.tpre.resize(16);
  memcpy(&t.tpre[0], &t.round, 8);
  memcpy(&t.tpre[8], &t.hq, 8);
  t.bp.resize(136);
  for (size_t j = 0; j < t.bp.size(); j++) t.bp[j] = (uint8_t)(r * 3 + j * 17 + 9);
  uint8_t qd[32], td[32], bd[32];
  hso_digest32(t.qp.data(), 40, qd);
  hso_digest32(t.tpre.data(), 16, td);
  hso_digest32(t.bp.data(), t.bp.size(), bd);
  // one signing pass: N authors over td, nv QC votes over qd, the Block author over bd
  const size_t n = (size_t)N + nv + 1;
  std::vector<uint32_t> key(n);
  std::vector<uint8_t> msgs(n * 32), sigs(n * 64);
  std::vector<uint64_t> off(n + 1);
  for (size_t i = 0; i < n; i++) {
    const bool author = i < (size_t)N, qc = !author && i < n - 1;
    key[i] = author ? (uint32_t)i : qc ? (uint32_t)(((i - N) * 7 + r) % N) : (uint32_t)((r + 1) % N);
    memcpy(&msgs[i * 32], author ? td : qc ? qd : bd, 32);
    off[i] = i * 32;
  }
  off[n] = n * 32;
  hso_sign_batch(k.seeds.data(), k.pks.data(), key.data(), msgs.data(), off.data(), n, ncpu(), sigs.data());
  t.asig.assign(sigs.begin(), sigs.begin() + (size_t)N * 64);
  t.qsig.assign(sigs.begin() + (size_t)N * 64, sigs.begin() + (n - 1) * 64);
  t.bsig.assign(sigs.end() - 64, sigs.end());
  t.bkey = key[n - 1];
  t.apk.resize((size_t)N * 32);
  t.qpk.resize((size_t)nv * 32);
  for (int i = 0; i < N; i++) {
    memcpy(&t.apk[(size_t)i * 32], &k.pks[(size_t)key[i] * 32], 32);
    if ((i * 37 + r * 11) % 100 == 0) t.asig[(size_t)i * 64 + (i + r) % 64] ^= 0x10;  // 1 % of the authors corrupted
  }
  for (int i = 0; i < nv; i++) memcpy(&t.qpk[(size_t)i * 32], &k.pks[(size_t)key[N + i] * 32], 32);
  auto oracle = [&](const std::vector<uint8_t> &sig, const std::vector<uint8_t> &pk, const uint8_t *d, size_t cnt, uint32_t mode) {
    std::vector<uint8_t> recs(cnt * 128);
    for (size_t i = 0; i < cnt; i++) {
      memcpy(&recs[i * 128], &sig[i * 64], 64);
      memcpy(&recs[i * 128 + 64], &pk[i * 32], 32);
      memcpy(&recs[i * 128 + 96], d, 32);
    }
    std::vector<uint32_t> w((cnt + 31) / 32);
    hso_verify_rec128_batch(recs.data(), cnt, mode, ncpu(), w.data());
    return w;
  };
  t.a_want = oracle(t.asig, t.apk, td, N, HS_MODE_STRICT);
  t.q_want = oracle(t.qsig, t.qpk, qd, nv, HS_MODE_BATCH_EQ);
  t.b_want = hso_verify_strict(t.bsig.data(), &k.pks[(size_t)t.bkey * 32], bd, 32) == 1;
}
// The round's N Timeouts through queue q from 16 threads (submit all, then wait for each); returns the verdict mismatches.
static int tc_timeouts(hs_queue *q, const tc_round &t, int N) {
  const int nv = N - (N - 1) / 3, nth = 16;
  std::atomic<int> mism{0};
  std::vector<std::thread> ts;
  for (int th = 0; th < nth; th++)
    ts.emplace_back([&, th] {
      std::vector<uint8_t> sig((size_t)(1 + nv) * 64), pk((size_t)(1 + nv) * 32), modes(1 + nv, HS_MODE_BATCH_EQ), pre(56);
      std::vector<uint32_t> midx(1 + nv, 1), bits((nv + 1 + 31) / 32);
      const uint64_t off[3] = {0, 16, 56};
      memcpy(&sig[64], t.qsig.data(), t.qsig.size());
      memcpy(&pk[32], t.qpk.data(), t.qpk.size());
      memcpy(pre.data(), t.tpre.data(), 16);
      memcpy(&pre[16], t.qp.data(), 40);
      modes[0] = HS_MODE_STRICT;
      midx[0] = 0;
      std::vector<std::pair<int, size_t>> tickets;
      for (int i = th; i < N; i += nth) {
        memcpy(sig.data(), &t.asig[(size_t)i * 64], 64);
        memcpy(pk.data(), &t.apk[(size_t)i * 32], 32);
        size_t ticket = 0;
        int rc;
        while ((rc = hs_queue_submit_msgs(q, pre.data(), off, 2, sig.data(), pk.data(), midx.data(), modes.data(), 1 + nv, nullptr, nullptr, &ticket)) ==
               HS_ERR_NOMEM)
          std::this_thread::yield();
        if (rc != HS_OK) {
          mism++;
          continue;
        }
        tickets.emplace_back(i, ticket);
      }
      for (auto &[i, ticket] : tickets) {
        if (hs_queue_wait(q, ticket, bits.data()) != HS_OK) {
          mism++;
          continue;
        }
        int m = bit(bits, 0) != bit(t.a_want, i);
        for (int v = 0; v < nv; v++) m += bit(bits, v + 1) != bit(t.q_want, v);
        mism += m;
      }
    });
  for (auto &th : ts) th.join();
  return mism.load();
}
static int tc_after_timeouts(hs_ctx *ctx, int N, int rounds, bool last) {
  const committee_keys k = make_keys(N, 47);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  const int nv = N - (N - 1) / 3;
  hs_queue *qs[2] = {nullptr, nullptr};  // arm (b): no signature cache, arm (c): with it
  for (int a = 0; a < 2; a++)
    if (hs_queue_create(ctx, 16384, &qs[a]) != HS_OK || hs_queue_cert_cache(qs[a], 64u << 20) != HS_OK) return 1;
  if (hs_queue_sig_cache(qs[1], 1u << 16) != HS_OK) return 1;
  uint64_t sig0[HS_QUEUE_SIG_STATS] = {}, tc_sig[2] = {0, 0}, blk_sig[2] = {0, 0};  // [probed, hits] of arm (c)'s TCs and Blocks
  hs_queue_sig_stats(qs[1], sig0);
  series lat[2][3];  // [TC, Block][arm]
  int mism[2][3] = {{0, 0, 0}, {0, 0, 0}}, to_mism = 0, errors = 0;
  tc_round t;
  for (int r = 0; r < rounds + 1; r++) {
    const bool timed = r >= 1;
    tc_make(k, r, t);
    // the TC: votes 0 .. nv - 1 are the first nv Timeouts' authors, each over its own copy of round || high_qc.round
    std::vector<uint8_t> tc_pre((size_t)nv * 16), tc_modes(nv, HS_MODE_STRICT);
    std::vector<uint64_t> tc_off(nv + 1), tc_hq(nv, t.hq);
    std::vector<uint32_t> tc_midx(nv), tc_want((nv + 31) / 32);
    for (int i = 0; i < nv; i++) {
      memcpy(&tc_pre[(size_t)i * 16], t.tpre.data(), 16);
      tc_off[i] = (uint64_t)i * 16;
      tc_midx[i] = (uint32_t)i;
      if (bit(t.a_want, i)) tc_want[i >> 5] |= 1u << (i & 31);
    }
    tc_off[nv] = (uint64_t)nv * 16;
    // the Block carrying the TC: author, the QC's votes, the TC's votes
    const size_t bn = 1 + 2 * (size_t)nv;
    std::vector<uint8_t> b_pre, b_sig(bn * 64), b_pk(bn * 32), b_modes(bn);
    std::vector<uint64_t> b_off{0};
    std::vector<uint32_t> b_midx(bn), b_want((bn + 31) / 32);
    auto add_pre = [&](const uint8_t *p, size_t len) {
      b_pre.insert(b_pre.end(), p, p + len);
      b_off.push_back(b_pre.size());
    };
    add_pre(t.bp.data(), t.bp.size());
    add_pre(t.qp.data(), 40);
    for (int i = 0; i < nv; i++) add_pre(t.tpre.data(), 16);
    memcpy(b_sig.data(), t.bsig.data(), 64);
    memcpy(b_pk.data(), &k.pks[(size_t)t.bkey * 32], 32);
    memcpy(&b_sig[64], t.qsig.data(), t.qsig.size());
    memcpy(&b_pk[32], t.qpk.data(), t.qpk.size());
    memcpy(&b_sig[(1 + (size_t)nv) * 64], t.asig.data(), (size_t)nv * 64);
    memcpy(&b_pk[(1 + (size_t)nv) * 32], t.apk.data(), (size_t)nv * 32);
    for (size_t i = 0; i < bn; i++) {
      const bool qc = i >= 1 && i <= (size_t)nv;
      b_modes[i] = qc ? HS_MODE_BATCH_EQ : HS_MODE_STRICT;
      b_midx[i] = i == 0 ? 0u : qc ? 1u : (uint32_t)(2 + i - 1 - nv);
      const bool w = i == 0 ? t.b_want : qc ? bit(t.q_want, (int)i - 1) : bit(t.a_want, (int)(i - 1 - nv));
      if (w) b_want[i >> 5] |= 1u << (i & 31);
    }
    for (int a = 0; a < 2; a++) to_mism += tc_timeouts(qs[a], t, N);
    for (int c = 0; c < 2; c++) {  // c = 0: the TC, 1: the Block
      const size_t n = c ? bn : (size_t)nv;
      std::vector<uint32_t> bits((n + 31) / 32);
      for (int a = 0; a < 3; a++) {
        uint64_t s0[HS_QUEUE_SIG_STATS] = {}, s1[HS_QUEUE_SIG_STATS] = {};
        if (a == 2) hs_queue_sig_stats(qs[1], s0);
        std::fill(bits.begin(), bits.end(), 0u);
        const auto t0 = clk::now();
        int rc;
        if (a == 0 && c == 0) {
          uint32_t tcb = 0;
          rc = hs_verify_tcs(ctx, &t.round, 1, t.apk.data(), nullptr, t.asig.data(), tc_hq.data(), std::vector<uint32_t>(n, 0).data(), n, bits.data(), &tcb);
        } else if (a == 0) {
          uint32_t gb = 0;
          rc = hs_verify_groups(ctx, b_pre.data(), b_off.data(), b_off.size() - 1, b_sig.data(), b_pk.data(), nullptr, b_midx.data(),
                                std::vector<uint32_t>(n, 0).data(), b_modes.data(), n, 1, bits.data(), &gb);
        } else {
          size_t ticket = 0;
          hs_queue *q = qs[a - 1];
          rc = c == 0 ? hs_queue_submit_msgs(q, tc_pre.data(), tc_off.data(), nv, t.asig.data(), t.apk.data(), tc_midx.data(), tc_modes.data(), n, nullptr,
                                             nullptr, &ticket)
                      : hs_queue_submit_msgs(q, b_pre.data(), b_off.data(), b_off.size() - 1, b_sig.data(), b_pk.data(), b_midx.data(), b_modes.data(), n,
                                             nullptr, nullptr, &ticket);
          if (rc == HS_OK) rc = hs_queue_wait(q, ticket, bits.data());
        }
        const double us = us_since(t0);
        errors += rc != HS_OK;
        if (a == 2) {
          hs_queue_sig_stats(qs[1], s1);
          if (timed) {
            uint64_t *d = c ? blk_sig : tc_sig;
            d[0] += s1[0] - s0[0];
            d[1] += s1[1] - s0[1];
          }
        }
        if (timed) {
          lat[c][a].v.push_back(us);
          const std::vector<uint32_t> &w = c ? b_want : tc_want;
          for (size_t i = 0; i < n; i++) mism[c][a] += bit(bits, (int)i) != bit(w, (int)i);
        }
      }
    }
  }
  printf("\"committee_%d\": {\"tc_votes\": %d, \"block_records\": %d, \"rounds\": %d, \"timeout_mismatches\": %d, \"errors\": %d, ", N, nv, 1 + 2 * nv, rounds,
         to_mism, errors);
  const char *cn[2] = {"tc", "block_with_tc"};
  const char *an[2][3] = {{"a_sync_verify_tcs", "b_queue_no_sig_cache", "c_queue_sig_cache"},
                          {"a_sync_verify_groups", "b_queue_no_sig_cache", "c_queue_sig_cache"}};
  for (int c = 0; c < 2; c++) {
    printf("\"%s\": {", cn[c]);
    for (int a = 0; a < 3; a++)
      printf("\"%s\": {\"p50_us\": %.1f, \"p99_us\": %.1f, \"mismatches\": %d}, ", an[c][a], lat[c][a].pct(0.5), lat[c][a].pct(0.99), mism[c][a]);
    const uint64_t *d = c ? blk_sig : tc_sig;
    printf("\"c_probed_per_round\": %.1f, \"c_hits_per_round\": %.1f}, ", (double)d[0] / rounds, (double)d[1] / rounds);
  }
  emit_sig_stats(qs[1], sig0);  // Timeouts, TCs and Blocks of every round, the warm-up round included
  printf("}%s", last ? "" : ", ");
  for (hs_queue *q : qs) hs_queue_destroy(q);
  int m = to_mism + errors;
  for (auto &row : mism)
    for (int x : row) m += x;
  return m;
}
static int run_tc_after_timeouts(hs_ctx *ctx, int rounds) {
  printf("\"tc_after_timeouts\": {\"gpu\": \"%s\", \"threads\": 16, \"ring_records\": 16384, \"sig_cache_entries\": %u, ", gpu_identity().c_str(), 1u << 16);
  int bad = 0;
  for (int N : {100, 1000, 4000}) bad += tc_after_timeouts(ctx, N, rounds, N == 4000);
  printf("}");
  return bad;
}

// ---- requests with keys outside the committee (alone with argv[3] = foreign_keys): the queue's slow path (hs_queue_generic off: the
// dispatcher thread verifies each such request synchronously) against its generic-key device path (on: k_queue_generic).
//   (a) no committee registered: a vote burst of N - f single-record requests from 16 threads, N = 100 and 1,000: the queue with the
//       option off, with it on, and the CPU oracle serially on one core;
//   (b) the committee registered: the same burst (every key registered) with ONE request by an unregistered key (1 or 500 records,
//       batch-eq) submitted once half the votes are in; p50 / p99 of the OTHER requests' latency with the option off and on, and
//       the foreign request's own latency.
// Every verdict, the foreign request's included, is checked against the oracle.
struct fk_req {
  clk::time_point *t0;
  double *lat;
  int *verdict;  // single-record request: its bit; the foreign group: 1 when every bit equals the oracle's, else 0
  const std::vector<int> *want;  // the foreign group's oracle verdicts (null for a vote)
};
static void on_fk(void *user, size_t, int status, const uint32_t *bitmap) {
  fk_req *r = (fk_req *)user;
  *r->lat = us_since(*r->t0);
  int v;
  if (status != HS_OK) v = -1;
  else if (!r->want) v = (int)(bitmap[0] & 1u);
  else {
    v = 1;
    for (size_t i = 0; i < r->want->size(); i++) v &= (int)((bitmap[i >> 5] >> (i & 31)) & 1u) == (*r->want)[i];
  }
  __atomic_store_n(r->verdict, v, __ATOMIC_RELEASE);
}
static int foreign_keys_arm(hs_ctx *ctx, int N, bool committee, int generic, int n_foreign, int bursts, series &burst, series &vote,
                            series &foreign, uint64_t gstats[HS_QUEUE_GENERIC_STATS], uint64_t qstats[HS_QUEUE_STATS], series *cpu) {
  const int f = (N - 1) / 3, nv = N - f, nth = 16;
  std::vector<uint8_t> seeds((size_t)N * 32), pks((size_t)N * 32), fseed(32), fpk(32);
  for (int i = 0; i < N; i++) {
    for (int j = 0; j < 32; j++) seeds[(size_t)i * 32 + j] = (uint8_t)(29 * i + 5 * j + 7 + (i >> 8));
    hso_keygen(&seeds[(size_t)i * 32], &pks[(size_t)i * 32]);
  }
  for (int j = 0; j < 32; j++) fseed[j] = (uint8_t)(201 + 3 * j);
  hso_keygen(fseed.data(), fpk.data());
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, pks.data(), committee ? N : 0, valid.data()) != HS_OK) return 1;
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 0, &q) != HS_OK || hs_queue_generic(q, generic) != HS_OK) return 1;
  int bad = 0;
  std::vector<hs_rec128> recs(nv), frecs(n_foreign);
  std::vector<uint8_t> fmodes(n_foreign, HS_MODE_BATCH_EQ);
  std::vector<int> want(nv), got(nv), fwant(n_foreign);
  std::vector<double> lat(nv);
  std::vector<fk_req> rq(nv);
  for (int r = 0; r < bursts + 3; r++) {
    const bool timed = r >= 3;
    uint8_t pre[40], d[32];
    for (int j = 0; j < 32; j++) pre[j] = (uint8_t)(r * 13 + j + 91 * generic);
    const uint64_t round = 5000 + (uint64_t)r;
    memcpy(pre + 32, &round, 8);
    hso_digest32(pre, 40, d);
    for (int i = 0; i < nv; i++) {
      const int k = (i * 7 + r) % N;
      hso_sign(&seeds[(size_t)k * 32], d, 32, recs[i].sig);
      memcpy(recs[i].pk, &pks[(size_t)k * 32], 32);
      memcpy(recs[i].msg, d, 32);
      if ((i * 37 + r * 11) % 100 == 0) recs[i].sig[(i + r) % 64] ^= 0x10;  // 1 % corrupted
    }
    for (int i = 0; i < n_foreign; i++) {  // the foreign request: its key signs distinct Digests; 1 % corrupted
      uint8_t m[8];
      memcpy(m, &i, 4);
      memcpy(m + 4, &r, 4);
      hso_digest32(m, 8, frecs[i].msg);
      hso_sign(fseed.data(), frecs[i].msg, 32, frecs[i].sig);
      memcpy(frecs[i].pk, fpk.data(), 32);
      if (i % 100 == 7) frecs[i].sig[40] ^= 1;
      fwant[i] = (hso_verify_flags(frecs[i].sig, frecs[i].pk, frecs[i].msg, 32) & HSO_EQ_OK) ? 1 : 0;
    }
    clk::time_point t0 = clk::now();
    for (int i = 0; i < nv; i++) {
      want[i] = hso_verify_strict(recs[i].sig, recs[i].pk, recs[i].msg, 32);
      lat[i] = us_since(t0);
    }
    if (timed && cpu) cpu->v.push_back(us_since(t0));
    std::atomic<int> go{0}, submitted{0};
    std::fill(got.begin(), got.end(), -2);
    int fgot = -2;
    double flat = 0;
    fk_req fr{&t0, &flat, &fgot, &fwant};
    std::vector<std::thread> ts;
    for (int t = 0; t < nth; t++)
      ts.emplace_back([&, t] {
        while (!go.load()) {
        }
        for (int i = t; i < nv; i += nth) {
          rq[i] = fk_req{&t0, &lat[i], &got[i], nullptr};
          int rc;
          while ((rc = hs_queue_submit(q, &recs[i], 1, HS_MODE_STRICT, on_fk, &rq[i], nullptr)) == HS_ERR_NOMEM) std::this_thread::yield();
          if (rc != HS_OK) bad++;
          submitted++;
        }
      });
    if (n_foreign)  // the foreign request, once half the votes are in
      ts.emplace_back([&] {
        while (submitted.load() < nv / 2) {
        }
        int rc;
        while ((rc = hs_queue_submit_group(q, frecs.data(), n_foreign, fmodes.data(), on_fk, &fr, nullptr)) == HS_ERR_NOMEM) std::this_thread::yield();
        if (rc != HS_OK) bad++;
      });
    t0 = clk::now();
    go = 1;
    for (auto &t : ts) t.join();
    for (int i = 0; i < nv; i++)
      while (__atomic_load_n(&got[i], __ATOMIC_ACQUIRE) == -2) std::this_thread::yield();
    if (n_foreign)
      while (__atomic_load_n(&fgot, __ATOMIC_ACQUIRE) == -2) std::this_thread::yield();
    for (int i = 0; i < nv; i++) bad += got[i] != want[i];
    if (n_foreign) bad += fgot != 1;
    if (timed) {
      burst.v.push_back(*std::max_element(lat.begin(), lat.end()));
      vote.v.insert(vote.v.end(), lat.begin(), lat.end());
      if (n_foreign) foreign.v.push_back(flat);
    }
  }
  hs_queue_generic_stats(q, gstats);
  hs_queue_stats(q, qstats);
  hs_queue_destroy(q);
  hs_committee_register(ctx, nullptr, 0, nullptr);
  return bad;
}
static int run_foreign_keys(hs_ctx *ctx, int bursts) {
  printf("\"foreign_keys\": {\"gpu\": \"%s\", \"threads\": 16, \"bursts\": %d, ", gpu_identity().c_str(), bursts);
  int bad = 0;
  const char *arm[2] = {"queue_generic_off", "queue_generic_on"};
  auto counters = [](const uint64_t *g, const uint64_t *s, int bursts) {
    printf("\"generic_launches_per_burst\": %.2f, \"generic_requests_per_burst\": %.1f, \"slow_requests_per_burst\": %.1f, \"small_launches_per_burst\": %.1f",
           (double)g[0] / (bursts + 3), (double)g[2] / (bursts + 3), (double)s[4] / (bursts + 3), (double)s[0] / (bursts + 3));
  };
  printf("\"no_committee\": {");
  for (int N : {100, 1000}) {
    printf("\"committee_%d\": {\"votes\": %d, ", N, N - (N - 1) / 3);
    series cpu;
    for (int g = 0; g < 2; g++) {
      series burst, vote, none;
      uint64_t gs[HS_QUEUE_GENERIC_STATS] = {}, qs[HS_QUEUE_STATS] = {};
      const int b = foreign_keys_arm(ctx, N, false, g, 0, bursts, burst, vote, none, gs, qs, g ? nullptr : &cpu);
      bad += b;
      printf("\"%s\": {\"burst_p50_us\": %.1f, \"burst_min_us\": %.1f, \"vote_p50_us\": %.1f, \"vote_p99_us\": %.1f, ", arm[g], burst.pct(0.5), burst.pct(0.0),
             vote.pct(0.5), vote.pct(0.99));
      counters(gs, qs, bursts);
      printf(", \"mismatches\": %d}, ", b);
    }
    printf("\"cpu_oracle_1core_serial\": {\"burst_p50_us\": %.1f}}%s", cpu.pct(0.5), N == 1000 ? "" : ", ");
  }
  printf("}, \"committee_registered_one_foreign_request\": {");
  for (int N : {100, 1000}) {
    printf("\"committee_%d\": {\"votes\": %d, ", N, N - (N - 1) / 3);
    for (int nf : {0, 1, 500}) {
      printf("\"foreign_records_%d\": {", nf);
      for (int g = 0; g < 2; g++) {
        series burst, vote, foreign;
        uint64_t gs[HS_QUEUE_GENERIC_STATS] = {}, qs[HS_QUEUE_STATS] = {};
        const int b = foreign_keys_arm(ctx, N, true, g, nf, bursts, burst, vote, foreign, gs, qs, nullptr);
        bad += b;
        printf("\"%s\": {\"other_requests_p50_us\": %.1f, \"other_requests_p99_us\": %.1f, \"burst_p50_us\": %.1f, \"foreign_request_p50_us\": %.1f, ", arm[g],
               vote.pct(0.5), vote.pct(0.99), burst.pct(0.5), foreign.pct(0.5));
        counters(gs, qs, bursts);
        printf(", \"mismatches\": %d}%s", b, g || nf == 0 ? "" : ", ");
        if (nf == 0) break;  // no foreign request: the option changes nothing
      }
      printf("}%s", nf == 500 ? "" : ", ");
    }
    printf("}%s", N == 1000 ? "" : ", ");
  }
  printf("}}");
  return bad;
}

// ---- the batch lane (alone with argv[3] = batch_lane): a whole hs_verify_groups pass as one queue request (hs_queue_submit_batch)
//   (a) replica_block, N = 1,000 .. 10,000: one Block (strict author over the Block preimage + N - f batch-eq QC votes over one
//       40-byte preimage, 1 % corrupted) through hs_queue_submit_batch (one group) + hs_queue_wait, hs_queue_submit_msgs +
//       hs_queue_wait, and the synchronous hs_verify_groups, one after another;
//   (b) block_during_burst, N = 1,000 and 10,000: the leader's vote burst from 16 threads with that Block arriving once half the
//       votes are in, on the lane or as hs_verify_groups from another thread; vote p50 / p99 and the Block's latency;
//   (c) view change, N = 100 / 1,000 / 4,000: the burst's N Timeouts collected into one batch (a group per author, one group for
//       the high_qc's votes) against Core::verify_timeouts' synchronous calls (hs_verify_tcs + one QC verify).
// Every verdict of every arm is checked against the oracle.
#define BL_MAX_ITEMS 32768
#define BL_MAX_BYTES (8u << 20)
static void bl_block(const committee_keys &k, int r, pre_cert &c) {  // make_pre_cert's Block without its TC
  make_pre_cert(k, r, true, c);
  const size_t n = 1 + (size_t)(k.N - (k.N - 1) / 3);
  c.off.resize(3);
  c.pre.resize(c.off[2]);
  c.sig.resize(n * 64);
  c.pk.resize(n * 32);
  c.midx.resize(n);
  c.modes.resize(n);
  c.want.resize((n + 31) / 32);
  if (n & 31) c.want.back() &= (1u << (n & 31)) - 1u;
}
static int bl_submit_wait(hs_queue *q, const pre_cert &c, uint32_t n_groups, const uint32_t *gidx, std::vector<uint32_t> &words) {
  const size_t n = c.midx.size();
  words.assign((n_groups + 31) / 32 + (n + 31) / 32, 0);
  size_t ticket = 0;
  int rc;
  while ((rc = hs_queue_submit_batch(q, c.pre.data(), c.off.data(), c.off.size() - 1, c.sig.data(), c.pk.data(), c.midx.data(), gidx, c.modes.data(), n,
                                     n_groups, nullptr, nullptr, &ticket)) == HS_ERR_NOMEM)
    std::this_thread::yield();
  return rc == HS_OK ? hs_queue_wait(q, ticket, words.data()) : rc;
}
static int bl_mismatch(const pre_cert &c, const uint32_t *item_bits) {
  int m = 0;
  for (size_t i = 0; i < c.midx.size(); i++) m += ((item_bits[i >> 5] >> (i & 31)) & 1u) != bit(c.want, (int)i);
  return m;
}
static int bl_replica_block(hs_ctx *ctx, hs_queue *q, int N, int blocks, bool last) {
  const committee_keys k = make_keys(N, 11);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  series lat[3];
  int mism[3] = {0, 0, 0}, bad = 0;
  pre_cert c;
  for (int r = 0; r < blocks + 3; r++) {
    const bool timed = r >= 3;
    bl_block(k, r, c);
    const size_t n = c.midx.size();
    std::vector<uint32_t> zeros(n, 0), words, bits((n + 31) / 32);
    for (int a = 0; a < 3; a++) {
      const auto t0 = clk::now();
      int rc;
      const uint32_t *items = bits.data();
      if (a == 0) {
        rc = bl_submit_wait(q, c, 1, zeros.data(), words);
        items = words.data() + 1;
      } else if (a == 1) {
        size_t ticket = 0;
        rc = hs_queue_submit_msgs(q, c.pre.data(), c.off.data(), c.off.size() - 1, c.sig.data(), c.pk.data(), c.midx.data(), c.modes.data(), n, nullptr, nullptr,
                                  &ticket);
        if (rc == HS_OK) rc = hs_queue_wait(q, ticket, bits.data());
      } else {
        uint32_t gb = 0;
        rc = hs_verify_groups(ctx, c.pre.data(), c.off.data(), c.off.size() - 1, c.sig.data(), c.pk.data(), nullptr, c.midx.data(), zeros.data(),
                              c.modes.data(), n, 1, bits.data(), &gb);
      }
      const double t = us_since(t0);
      bad += rc != HS_OK;
      if (timed) {
        lat[a].v.push_back(t);
        mism[a] += bl_mismatch(c, items);
      }
    }
  }
  printf("\"committee_%d\": {\"records\": %zu, \"blocks\": %d, ", N, c.midx.size(), blocks);
  const char *names[3] = {"a_submit_batch", "b_submit_msgs", "c_sync_verify_groups"};
  for (int a = 0; a < 3; a++) printf("\"%s\": {\"p50_us\": %.1f, \"p99_us\": %.1f, \"mismatches\": %d}, ", names[a], lat[a].pct(0.5), lat[a].pct(0.99), mism[a]);
  printf("\"errors\": %d}%s", bad, last ? "" : ", ");
  return mism[0] + mism[1] + mism[2] + bad;
}
static int bl_block_during_burst(hs_ctx *ctx, int N, int bursts, bool last) {
  const int f = (N - 1) / 3, nv = N - f, nth = 16;
  const committee_keys k = make_keys(N, 23);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 16384, &q) != HS_OK || hs_queue_batch(q, BL_MAX_ITEMS, BL_MAX_BYTES) != HS_OK) return 1;
  burst_arm arm[2];
  series blk[2];
  int blk_bad[2] = {0, 0};
  std::vector<hs_rec128> votes(nv);
  std::vector<int> want(nv), got(nv);
  std::vector<double> lat(nv);
  std::vector<burst_vote> bv(nv);
  pre_cert c;
  for (int r = 0; r < bursts + 3; r++) {
    const bool timed = r >= 3;
    bl_block(k, 1000 + r, c);  // the replica's Block (another round's certificate)
    const size_t nb = c.midx.size();
    std::vector<uint32_t> zeros(nb, 0);
    uint8_t pre[40], d[32];
    for (int j = 0; j < 32; j++) pre[j] = (uint8_t)(r * 13 + j);
    const uint64_t round = 1000 + (uint64_t)r;
    memcpy(pre + 32, &round, 8);
    hso_digest32(pre, 40, d);
    for (int i = 0; i < nv; i++) {
      const int kk = (i * 7 + r) % N;
      hso_sign(&k.seeds[(size_t)kk * 32], d, 32, votes[i].sig);
      memcpy(votes[i].pk, &k.pks[(size_t)kk * 32], 32);
      memcpy(votes[i].msg, d, 32);
      if ((i * 37 + r * 11) % 100 == 0) votes[i].sig[(i + r) % 64] ^= 0x10;
    }
    std::vector<uint32_t> wb((nv + 31) / 32);
    hso_verify_rec128_batch((const uint8_t *)votes.data(), nv, 0, ncpu(), wb.data());
    for (int i = 0; i < nv; i++) want[i] = bit(wb, i);
    for (int a = 0; a < 2; a++) {  // a = 0: the Block on the batch lane; a = 1: hs_verify_groups on another thread
      std::atomic<int> go{0}, submitted{0}, bad{0}, blk_ok{0};
      double blk_lat = 0;
      std::vector<uint32_t> words, items((nb + 31) / 32);
      std::vector<std::thread> ts;
      std::fill(got.begin(), got.end(), -2);
      clk::time_point t0;
      for (int t = 0; t < nth; t++)
        ts.emplace_back([&, t] {
          while (!go.load()) {
          }
          for (int i = t; i < nv; i += nth) {
            bv[i] = burst_vote{t0, &lat[i], &got[i]};
            int rc;
            while ((rc = hs_queue_submit(q, &votes[i], 1, HS_MODE_STRICT, on_vote, &bv[i], nullptr)) == HS_ERR_NOMEM) std::this_thread::yield();
            if (rc != HS_OK) bad++;
            submitted++;
          }
        });
      ts.emplace_back([&] {  // the replica's connection task: its Block arrives when half the votes are in
        while (submitted.load() < nv / 2) {
        }
        const auto tb = clk::now();
        int rc;
        if (a == 0) {
          rc = bl_submit_wait(q, c, 1, zeros.data(), words);
          if (rc == HS_OK) std::copy(words.begin() + 1, words.end(), items.begin());
        } else {
          uint32_t gb = 0;
          rc = hs_verify_groups(ctx, c.pre.data(), c.off.data(), c.off.size() - 1, c.sig.data(), c.pk.data(), nullptr, c.midx.data(), zeros.data(),
                                c.modes.data(), nb, 1, items.data(), &gb);
        }
        blk_lat = us_since(tb);
        blk_ok = rc == HS_OK;
      });
      t0 = clk::now();
      go = 1;
      for (auto &t : ts) t.join();
      for (int i = 0; i < nv; i++)
        while (__atomic_load_n(&got[i], __ATOMIC_ACQUIRE) == -2) std::this_thread::yield();
      if (timed) {
        arm[a].total.v.push_back(*std::max_element(lat.begin(), lat.end()));
        arm[a].vote.v.insert(arm[a].vote.v.end(), lat.begin(), lat.end());
        for (int i = 0; i < nv; i++) arm[a].mismatches += got[i] != want[i];
        arm[a].mismatches += bad.load();
        blk[a].v.push_back(blk_lat);
        blk_bad[a] += (blk_ok.load() != 1) + bl_mismatch(c, items.data());
      }
    }
  }
  printf("\"committee_%d\": {\"votes\": %d, \"block_records\": %zu, \"bursts\": %d, ", N, nv, c.midx.size(), bursts);
  const char *names[2] = {"block_via_submit_batch", "block_via_sync_verify_groups_other_thread"};
  for (int a = 0; a < 2; a++) {
    printf("\"%s\": {\"block_p50_us\": %.1f, \"block_p99_us\": %.1f, \"block_mismatches\": %d, ", names[a], blk[a].pct(0.5), blk[a].pct(0.99), blk_bad[a]);
    arm[a].emit("votes", bursts, true);
    printf("}%s", a == 0 ? ", " : "");
  }
  printf("}%s", last ? "" : ", ");
  hs_queue_destroy(q);
  return arm[0].mismatches + arm[1].mismatches + blk_bad[0] + blk_bad[1];
}
// The view-change burst as one batch: group i = Timeout i's author (strict, over round || high_qc.round), group N = the high_qc's
// votes (batch-eq, over hash || round).
static int bl_view_change(hs_ctx *ctx, hs_queue *q, int N, int bursts, bool last) {
  const committee_keys k = make_keys(N, 41);
  std::vector<uint32_t> valid((N + 31) / 32);
  if (hs_committee_register(ctx, k.pks.data(), N, valid.data()) != HS_OK) return 1;
  series lat;
  vc_arm sync_arm, scratch;
  int mism = 0, bad = 0;
  vc_burst v;
  for (int b = 0; b < bursts + 2; b++) {
    const bool timed = b >= 2;
    vc_make(k, b, false, v);
    pre_cert c;  // the collected burst in hs_verify_groups' arrays
    c.pre.resize(56);
    memcpy(c.pre.data(), &v.round, 8);
    memcpy(c.pre.data() + 8, &v.hq, 8);
    memcpy(c.pre.data() + 16, v.qc[0].pre, 40);
    c.off = {0, 16, 56};
    const size_t n = (size_t)N + v.nv;
    std::vector<uint32_t> gidx(n);
    c.sig = v.a_sig;
    c.sig.insert(c.sig.end(), v.qc[0].sig.begin(), v.qc[0].sig.end());
    c.pk = v.a_pk;
    c.pk.insert(c.pk.end(), v.qc[0].pk.begin(), v.qc[0].pk.end());
    c.midx.assign(n, 1);
    c.modes.assign(n, HS_MODE_BATCH_EQ);
    c.want.assign((n + 31) / 32, 0);
    for (size_t i = 0; i < n; i++) {
      const bool author = i < (size_t)N;
      gidx[i] = author ? (uint32_t)i : (uint32_t)N;
      if (author) c.midx[i] = 0, c.modes[i] = HS_MODE_STRICT;
      if (author ? bit(v.a_want, (int)i) : bit(v.qc[0].want, (int)(i - N))) c.want[i >> 5] |= 1u << (i & 31);
    }
    std::vector<uint32_t> words;
    const auto t0 = clk::now();
    bad += bl_submit_wait(q, c, (uint32_t)N + 1, gidx.data(), words) != HS_OK;
    const double t = us_since(t0);
    const double ts = vc_sync_burst(ctx, v, timed ? sync_arm : scratch);
    if (timed) {
      lat.v.push_back(t);
      sync_arm.t.v.push_back(ts);
      mism += bl_mismatch(c, words.data() + (N + 1 + 31) / 32);
    }
  }
  bad += scratch.mismatches + scratch.errors;
  printf("\"committee_%d\": {\"timeouts_per_burst\": %d, \"batch_items\": %d, \"bursts\": %d, \"a_submit_batch\": {\"burst_p50_us\": %.1f, \"burst_p99_us\": %.1f, "
         "\"mismatches\": %d}, \"b_sync_verify_tcs_plus_qc\": {\"burst_p50_us\": %.1f, \"burst_p99_us\": %.1f, \"mismatches\": %d}, \"errors\": %d}%s",
         N, N, N + v.nv, bursts, lat.pct(0.5), lat.pct(0.99), mism, sync_arm.t.pct(0.5), sync_arm.t.pct(0.99), sync_arm.mismatches, bad + sync_arm.errors,
         last ? "" : ", ");
  return mism + bad + sync_arm.mismatches + sync_arm.errors;
}
static int run_batch_lane(hs_ctx *ctx, int reps) {
  printf("\"batch_lane\": {\"gpu\": \"%s\", \"max_items\": %d, \"max_bytes\": %u, \"replica_block\": {\"ring_records\": 16384, ", gpu_identity().c_str(),
         BL_MAX_ITEMS, BL_MAX_BYTES);
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 16384, &q) != HS_OK || hs_queue_batch(q, BL_MAX_ITEMS, BL_MAX_BYTES) != HS_OK) return 1;
  int bad = 0;
  for (int N : {1000, 1500, 3000, 6000, 10000}) bad += bl_replica_block(ctx, q, N, reps, N == 10000);
  printf("}, \"block_during_burst\": {\"threads\": 16, ");
  bad += bl_block_during_burst(ctx, 1000, reps, false);
  bad += bl_block_during_burst(ctx, 10000, reps, true);
  printf("}, \"view_change\": {");
  for (int N : {100, 1000, 4000}) bad += bl_view_change(ctx, q, N, reps, N == 4000);
  printf("}, ");
  uint64_t s[HS_QUEUE_BATCH_STATS] = {};
  hs_queue_batch_stats(q, s);
  printf("\"batch_stats\": {\"passes\": %llu, \"items\": %llu, \"groups\": %llu, \"preimage_bytes\": %llu, \"outside_committee\": %llu}}",
         (unsigned long long)s[0], (unsigned long long)s[1], (unsigned long long)s[2], (unsigned long long)s[3], (unsigned long long)s[4]);
  hs_queue_destroy(q);
  return bad;
}

int main(int argc, char **argv) {
  const int rounds = argc > 1 ? atoi(argv[1]) : 1000;
  hs_ctx *ctx = nullptr;
  if (hs_ctx_create(&ctx, 0, 0) != HS_OK) {
    fprintf(stderr, "hs_ctx_create failed (no GPU?)\n");
    return 1;
  }
  if (argc > 3 && strcmp(argv[3], "certificate_preimages") == 0) {
    printf("{");
    const int bad = run_certificate_preimages(ctx, argc > 2 ? atoi(argv[2]) : 20);
    printf("}\n");
    hs_ctx_destroy(ctx);
    return bad ? 9 : 0;
  }
  if (argc > 3 && strcmp(argv[3], "foreign_keys") == 0) {
    printf("{");
    const int bad = run_foreign_keys(ctx, argc > 2 ? atoi(argv[2]) : 10);
    printf("}\n");
    hs_ctx_destroy(ctx);
    return bad ? 9 : 0;
  }
  if (argc > 3 && strcmp(argv[3], "batch_lane") == 0) {
    printf("{");
    const int bad = run_batch_lane(ctx, argc > 2 ? atoi(argv[2]) : 20);
    printf("}\n");
    hs_ctx_destroy(ctx);
    return bad ? 9 : 0;
  }
  if (argc > 3 && strcmp(argv[3], "view_change") == 0) {
    printf("{");
    const int bad = run_view_change(ctx, argc > 2 ? atoi(argv[2]) : 10);
    printf("}\n");
    hs_ctx_destroy(ctx);
    return bad ? 9 : 0;
  }
  if (argc > 3 && (strcmp(argv[3], "tc_after_timeouts") == 0 || strcmp(argv[3], "sig_cache_cost") == 0)) {
    printf("{");
    const bool tc = strcmp(argv[3], "tc_after_timeouts") == 0;
    const int bad = tc ? run_tc_after_timeouts(ctx, argc > 2 ? atoi(argv[2]) : 10) : run_sig_cache_cost(ctx, argc > 2 ? atoi(argv[2]) : 20);
    printf("}\n");
    hs_ctx_destroy(ctx);
    return bad ? 9 : 0;
  }
  uint8_t seeds[4][32], pks[4][32];
  for (int i = 0; i < 4; i++) {
    for (int j = 0; j < 32; j++) seeds[i][j] = (uint8_t)(17 * i + 3 * j + 1);
    hso_keygen(seeds[i], pks[i]);
  }
  uint32_t valid = 0;
  if (hs_committee_register(ctx, &pks[0][0], 4, &valid) != HS_OK || valid != 0xf) return 2;
  // one serialized MempoolMessage::Batch (bincode: u32 tag, u64 count, per tx u64 len + bytes), 29 x 512 B
  const int tx = 512, per_batch = 15000 / tx;
  std::vector<uint8_t> batch(12 + (size_t)per_batch * (8 + tx));
  memset(batch.data(), 0, batch.size());
  uint64_t cnt = per_batch;
  memcpy(batch.data() + 4, &cnt, 8);
  for (int t = 0; t < per_batch; t++) {
    uint64_t l = tx;
    uint8_t *p = batch.data() + 12 + (size_t)t * (8 + tx);
    memcpy(p, &l, 8);
    for (int j = 0; j < tx; j++) p[8 + j] = (uint8_t)(t * 31 + j * 7);
  }
  std::vector<uint8_t> two(batch.size() * 2);
  memcpy(two.data(), batch.data(), batch.size());
  memcpy(two.data() + batch.size(), batch.data(), batch.size());
  two[batch.size() + 20] ^= 1;
  const uint64_t off1[2] = {0, batch.size()}, off2[3] = {0, batch.size(), 2 * batch.size()};
  series g_d1, g_d2, g_v1, g_b3, g_v3, c_d1, c_d2, c_v1, c_b3, c_v3;
  uint8_t dig[64], want[64];
  int bad = 0;
  for (int r = 0; r < rounds + 20; r++) {
    const bool timed = r >= 20;  // warm-up rounds
    uint8_t blk[40], bd[32];
    memset(blk, 0, sizeof(blk));
    memcpy(blk, &r, 4);
    hso_digest32(blk, 40, bd);
    hs_rec128 recs[4];
    hs_vote votes[3];
    for (int i = 0; i < 4; i++) {
      hso_sign(seeds[i], bd, 32, recs[i].sig);
      memcpy(recs[i].pk, pks[i], 32);
      memcpy(recs[i].msg, bd, 32);
    }
    for (int i = 0; i < 3; i++) {
      memcpy(votes[i].pk, pks[i + 1], 32);
      memcpy(votes[i].sig, recs[i + 1].sig, 64);
    }
    if (r % 7 == 3) recs[2].sig[9] ^= 4;  // an invalid vote now and then: verdicts must follow
    uint32_t bm = 0;
    int all_ok = 0;
    auto t0 = clk::now();
    if (hs_digest32_batch(ctx, batch.data(), off1, 1, dig) != HS_OK) return 3;
    if (timed) g_d1.v.push_back(us_since(t0));
    t0 = clk::now();
    if (hs_digest32_batch(ctx, two.data(), off2, 2, dig) != HS_OK) return 3;  // the ~1.7 batches of a round submitted together
    if (timed) g_d2.v.push_back(us_since(t0));
    t0 = clk::now();
    if (hs_verify_strict_batch(ctx, &recs[0], 1, &bm) != HS_OK) return 4;
    if (timed) g_v1.v.push_back(us_since(t0));
    bad += (bm & 1) != 1;
    t0 = clk::now();
    if (hs_verify_batch_shared_msg(ctx, bd, votes, 3, &all_ok, nullptr) != HS_OK) return 5;
    if (timed) g_b3.v.push_back(us_since(t0));
    bad += all_ok != 1;
    t0 = clk::now();
    if (hs_verify_strict_batch(ctx, &recs[1], 3, &bm) != HS_OK) return 6;
    if (timed) g_v3.v.push_back(us_since(t0));
    bad += bm != ((r % 7 == 3) ? 0x5u : 0x7u);
    // CPU column (oracle, one core)
    t0 = clk::now();
    hso_digest32(batch.data(), batch.size(), want);
    if (timed) c_d1.v.push_back(us_since(t0));
    t0 = clk::now();
    hso_digest32(two.data(), batch.size(), want);
    hso_digest32(two.data() + batch.size(), batch.size(), want + 32);
    if (timed) c_d2.v.push_back(us_since(t0));
    bad += memcmp(want, dig, 64) != 0;
    t0 = clk::now();
    int ok = hso_verify_strict(recs[0].sig, recs[0].pk, recs[0].msg, 32);
    if (timed) c_v1.v.push_back(us_since(t0));
    bad += ok != 1;
    t0 = clk::now();
    ok = hso_verify_batch_shared_msg(bd, (const uint8_t *)votes, 3, 1, nullptr);
    if (timed) c_b3.v.push_back(us_since(t0));
    t0 = clk::now();
    for (int i = 1; i < 4; i++) ok += hso_verify_strict(recs[i].sig, recs[i].pk, recs[i].msg, 32);
    if (timed) c_v3.v.push_back(us_since(t0));
  }
  const double per_round = g_d2.mean() + g_v1.mean() + g_b3.mean() + g_v3.mean();
  const double per_round_cpu = c_d2.mean() + c_v1.mean() + c_b3.mean() + c_v3.mean();
  printf("{\"what\": \"replay of the per-node crypto call stream of fab local @ 50k tx/s, 512 B tx, 4 nodes through the C ABI (not a fab run)\", \"rounds\": %d, "
         "\"mismatches\": %d, \"calls\": {",
         rounds, bad);
  emit("digest_one_15kB_batch", g_d1, c_d1, false);
  emit("digest_two_15kB_batches_one_call", g_d2, c_d2, false);
  emit("verify_strict_1", g_v1, c_v1, false);
  emit("verify_batch_3", g_b3, c_b3, false);
  emit("verify_strict_3", g_v3, c_v3, true);
  printf("}, \"crypto_us_per_round_gpu\": %.1f, \"rounds_per_s_sustainable_single_caller_gpu\": %.0f, \"crypto_us_per_round_cpu_oracle_1core\": %.1f, "
         "\"kernel_launches\": %llu, ",
         per_round, 1e6 / per_round, per_round_cpu, (unsigned long long)hs_kernel_launches(ctx));
  const int bursts = argc > 2 ? atoi(argv[2]) : 20;
  printf("\"leader_vote_burst\": {\"gpu\": \"%s\", \"threads\": 16, ", gpu_identity().c_str());
  int burst_bad = 0;
  for (int N : {4, 100, 1000}) burst_bad += vote_burst(ctx, N, bursts, N == 1000);
  printf("}, \"replica_block\": {\"gpu\": \"%s\", \"ring_records\": 16384, ", gpu_identity().c_str());
  hs_queue *q = nullptr;
  if (hs_queue_create(ctx, 16384, &q) != HS_OK) return 1;
  for (int N : {4, 100, 250, 500, 750, 1000, 1500, 3000, 6000, 10000}) burst_bad += replica_block(ctx, q, N, bursts, N == 10000);
  hs_queue_destroy(q);
  printf("}, \"block_during_burst\": {\"gpu\": \"%s\", \"threads\": 16, ", gpu_identity().c_str());
  burst_bad += block_during_burst(ctx, 1000, 0, bursts, false);
  burst_bad += block_during_burst(ctx, 10000, 16384, bursts, true);
  printf("}, ");
  burst_bad += run_certificate_preimages(ctx, bursts);
  printf(", ");
  burst_bad += run_view_change(ctx, bursts);
  printf("}\n");
  hs_ctx_destroy(ctx);
  return (bad || burst_bad) ? 9 : 0;
}
