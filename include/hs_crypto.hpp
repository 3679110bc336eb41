// hs_crypto.hpp — header-only C++ mirror of asonnino/hotstuff's `crypto` crate surface over the C ABI (hs_crypto.h).
//
// The reference is compiled Rust (crypto/src/lib.rs); with no Rust toolchain in the build image, this is the compiled-language
// host side above the ABI: same type names, argument meaning and error behaviour as the crate —
//   Digest (lib.rs:22), PublicKey (lib.rs:66), Signature{verify (lib.rs:200-204), verify_batch (lib.rs:206-219)}, CryptoError (lib.rs:18).
// Signing (Signature::new, SignatureService) stays on the CPU in the reference node and is not part of the GPU path.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <future>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "hs_crypto.h"

namespace hs {

// `CryptoError = ed25519::Error`: opaque, only Ok/Err is observable (consensus maps it to InvalidSignature, error.rs:39).
struct CryptoError : std::runtime_error {
  CryptoError() : std::runtime_error("signature error") {}
};
// Engine failure (CUDA error / bad argument): NOT a verdict.  Callers treat it as reject (core.rs:434-439 drops the message).
struct EngineError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

class VerifyQueue;

class Engine {
 public:
  explicit Engine(int device = 0, uint32_t flags = 0) {
    if (hs_ctx_create(&ctx_, device, flags) != HS_OK) throw EngineError("hs_ctx_create failed (no GPU?) — there is no CPU fallback");
  }
  // A non-owning Engine on a context another object owns (MultiEngine::member): the destructor leaves the context alone.
  struct Borrowed {};
  Engine(hs_ctx *ctx, Borrowed) : ctx_(ctx), owned_(false) {}
  ~Engine() {
    if (owned_) hs_ctx_destroy(ctx_);
  }
  Engine(const Engine &) = delete;
  Engine &operator=(const Engine &) = delete;
  hs_ctx *raw() const { return ctx_; }
  void check(int rc, const char *what) const {
    if (rc != HS_OK) throw EngineError(std::string(what) + ": " + hs_last_error(ctx_));
  }
  // Known-answer self-test of every device path at this context's geometry (hs_self_test, built-in set, key_bits 0 = the window in
  // use): 0 when every answer is right, else the HS_SELFTEST_* bits of the failing paths (error() names the first mismatch).  Throws
  // EngineError when the test cannot run (no device memory for its scratch tables, CUDA error).
  uint32_t self_test(int key_bits = 0) const {
    uint32_t failed = 0;
    const int rc = hs_self_test(ctx_, key_bits, nullptr, nullptr, 0, &failed);
    if (rc != HS_ERR_SELFTEST) check(rc, "hs_self_test");
    return failed;
  }
  // Key slots in use (hs_key_slots): the committee's, spare slots taken by updates included, or the key cache's learned keys.
  size_t key_slots() const { return hs_key_slots(ctx_); }
  // Audit of the live key tables (hs_table_audit): 0 when every check passes, else the HS_AUDIT_* bits (error() names the first
  // finding).  expect: the node's index -> key map (key_slots() entries, nullptr = the engine against itself); live: one bit per slot
  // expected live (nullptr = all); slot_bits (nullable) receives each slot's HS_AUDIT_* bits.  Throws EngineError on a bad argument,
  // tables that changed during the audit (call again), no device memory or a CUDA error.
  uint32_t table_audit(const std::vector<std::array<uint8_t, 32>> *expect = nullptr, const std::vector<uint32_t> *live = nullptr,
                       std::vector<uint8_t> *slot_bits = nullptr) const {
    const size_t n = expect ? expect->size() : key_slots();
    if (live && live->size() < (n + 31) / 32) throw EngineError("table_audit: live bitmap shorter than the slots");
    std::vector<uint8_t> bits(n);
    uint32_t failed = 0;
    const int rc = hs_table_audit(ctx_, expect && n ? expect->front().data() : nullptr, live && !live->empty() ? live->data() : nullptr, n,
                                  bits.data(), &failed);
    if (rc != HS_ERR_SELFTEST) check(rc, "hs_table_audit");
    if (slot_bits) *slot_bits = std::move(bits);
    return failed;
  }
  // Repair of what the audit finds (hs_table_repair), from the same authority: `expect` / `live` as for table_audit, else the engine's
  // mirror.  Returns the classes the final audit still finds (0: repaired, or nothing was wrong); found receives the classes the first
  // audit found, slot_bits (nullable) its per-slot bits.  Throws EngineError as table_audit does.
  uint32_t table_repair(const std::vector<std::array<uint8_t, 32>> *expect = nullptr, const std::vector<uint32_t> *live = nullptr,
                        uint32_t *found = nullptr, std::vector<uint8_t> *slot_bits = nullptr) const {
    const size_t n = expect ? expect->size() : key_slots();
    if (live && live->size() < (n + 31) / 32) throw EngineError("table_repair: live bitmap shorter than the slots");
    std::vector<uint8_t> bits(n);
    uint32_t f = 0, failed = 0;
    const int rc = hs_table_repair(ctx_, expect && n ? expect->front().data() : nullptr, live && !live->empty() ? live->data() : nullptr, n,
                                   bits.data(), &f, &failed);
    if (rc != HS_ERR_SELFTEST) check(rc, "hs_table_repair");
    if (found) *found = f;
    if (slot_bits) *slot_bits = std::move(bits);
    return failed;
  }
  // Mend of corrupt comb-table entries in place (hs_table_mend): no drain, no slot out of service.  Arguments as for table_repair.
  // Returns the classes left for table_repair (0: everything mended, or nothing was wrong; KEY, FLAG and LOOKUP are always left); found
  // receives the classes the audit found, slot_bits (nullable) its per-slot bits.  Throws EngineError as table_audit does.
  uint32_t table_mend(const std::vector<std::array<uint8_t, 32>> *expect = nullptr, const std::vector<uint32_t> *live = nullptr,
                      uint32_t *found = nullptr, std::vector<uint8_t> *slot_bits = nullptr) const {
    const size_t n = expect ? expect->size() : key_slots();
    if (live && live->size() < (n + 31) / 32) throw EngineError("table_mend: live bitmap shorter than the slots");
    std::vector<uint8_t> bits(n);
    uint32_t f = 0, left = 0;
    const int rc = hs_table_mend(ctx_, expect && n ? expect->front().data() : nullptr, live && !live->empty() ? live->data() : nullptr, n,
                                 bits.data(), &f, &left);
    if (rc != HS_ERR_SELFTEST) check(rc, "hs_table_mend");
    if (found) *found = f;
    if (slot_bits) *slot_bits = std::move(bits);
    return left;
  }
  // calls, windows recomputed, entries rewritten, windows left, slots left to repair, cache flushes (hs_table_mend_stats).
  std::array<uint64_t, HS_MEND_STATS> mend_stats() const {
    std::array<uint64_t, HS_MEND_STATS> s{};
    check(hs_table_mend_stats(ctx_, s.data()), "hs_table_mend_stats");
    return s;
  }
  // on: a scrub tick whose findings can all be mended mends them instead of repairing them (hs_scrub_mend).
  void scrub_mend(bool on) const { check(hs_scrub_mend(ctx_, on ? 1 : 0), "hs_scrub_mend"); }
  // The engine-owned scrub (hs_scrub_start): every period_us a thread audits the next slots_per_tick slots in service and
  // base_entries_per_tick base-point entries against `expect` / `live` (as for table_audit; the engine copies them), repairs what it
  // finds and calls cb (nullable) once per tick that found anything, on its thread.  After a committee change it pauses until
  // scrub_set_map.  Throws EngineError when a scrub already runs or the map breaks the audit's rules.
  void scrub_start(const std::vector<std::array<uint8_t, 32>> *expect, const std::vector<uint32_t> *live, uint32_t period_us,
                   uint32_t slots_per_tick, uint32_t base_entries_per_tick, hs_scrub_cb *cb = nullptr, void *user = nullptr) const {
    const size_t n = expect ? expect->size() : key_slots();
    if (live && live->size() < (n + 31) / 32) throw EngineError("scrub_start: live bitmap shorter than the slots");
    check(hs_scrub_start(ctx_, expect && n ? expect->front().data() : nullptr, live && !live->empty() ? live->data() : nullptr, n, period_us,
                         slots_per_tick, base_entries_per_tick, cb, user),
          "hs_scrub_start");
  }
  // The map of the slots after a committee change (hs_scrub_set_map): the paused scrub resumes with a new pass.
  void scrub_set_map(const std::vector<std::array<uint8_t, 32>> *expect = nullptr, const std::vector<uint32_t> *live = nullptr) const {
    const size_t n = expect ? expect->size() : key_slots();
    if (live && live->size() < (n + 31) / 32) throw EngineError("scrub_set_map: live bitmap shorter than the slots");
    check(hs_scrub_set_map(ctx_, expect && n ? expect->front().data() : nullptr, live && !live->empty() ? live->data() : nullptr, n),
          "hs_scrub_set_map");
  }
  // Stops the scrub and joins its thread (hs_scrub_stop); a no-op when none runs.  Not from the scrub's callback.
  void scrub_stop() const { check(hs_scrub_stop(ctx_), "hs_scrub_stop"); }
  // passes, slots audited, base entries audited, ticks, findings, slots repaired, failed repairs, ticks paused (hs_scrub_stats).
  std::array<uint64_t, HS_SCRUB_STATS> scrub_stats() const {
    std::array<uint64_t, HS_SCRUB_STATS> s{};
    check(hs_scrub_stats(ctx_, s.data()), "hs_scrub_stats");
    return s;
  }
  // Attaches q (a queue of this engine) to the scrub (hs_scrub_sig_cache): every tick also audits the next buckets_per_tick buckets of
  // its signature cache, and a tick that corrected an entry calls back with HS_AUDIT_SIGCACHE in found.  nullptr detaches.
  inline void scrub_sig_cache(const VerifyQueue *q, uint32_t buckets_per_tick = 512) const;
  // Table-free re-check of n records (hs_explain_rec128): one byte of HS_WHY_* bits per record, one bit per failed check.  Strict
  // verdict 1 <=> 0; batch-eq verdict 1 <=> no bit outside HS_WHY_A_SMALL | HS_WHY_R_SMALL.  Throws EngineError on a CUDA error.
  std::vector<uint8_t> explain(const hs_rec128 *recs, size_t n) const {
    std::vector<uint8_t> why(n);
    check(hs_explain_rec128(ctx_, recs, n, why.data()), "hs_explain_rec128");
    return why;
  }
  // The same re-check for the rejected items of a device-resident pass (hs_explain_groups_dev), enqueued on `stream` (a cudaStream_t)
  // with every array in device memory: the pass's arrays with key bytes in d_pk, its item bitmap, and max_explain (0 = every rejected
  // item).  d_why receives n_items bytes (HS_WHY_NOT_EXAMINED for an item not examined), d_out HS_EXPLAIN_DEV_OUT words: items whose
  // bit is 0, items examined, engine faults, the lowest faulting index (0xffffffff: none).  Throws EngineError when nothing was enqueued.
  void explain_groups_dev(const void *d_preimages, const void *d_pre_off, size_t n_msgs, const void *d_sig, const void *d_pk, const void *d_msg_idx,
                          const void *d_mode_or_null, const void *d_item_bitmap, size_t n_items, size_t max_explain, void *d_why, void *d_out,
                          void *stream) const {
    check(hs_explain_groups_dev(ctx_, d_preimages, d_pre_off, n_msgs, d_sig, d_pk, d_msg_idx, d_mode_or_null, d_item_bitmap, n_items, max_explain,
                                d_why, d_out, stream),
          "hs_explain_groups_dev");
  }
  // Staged committee change (hs_committee_stage): the added keys' tables are built and proved off the verify path and nothing changes
  // for verification until committee_commit.  Returns the indices the added keys will have: stage + commit leaves the engine as
  // hs_committee_update(add) then hs_committee_update(remove) would.  Throws EngineError on any failure (HS_ERR_NOMEM: too few free and
  // spare slots, use hs_committee_update).
  std::vector<uint32_t> committee_stage(const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove) const {
    std::vector<uint32_t> idx(n_add);
    check(hs_committee_stage(ctx_, add_pks, n_add, remove_idx, n_remove, idx.data()), "hs_committee_stage");
    return idx;
  }
  void committee_commit() const { check(hs_committee_commit(ctx_), "hs_committee_commit"); }
  void committee_discard() const { check(hs_committee_discard(ctx_), "hs_committee_discard"); }
  // A whole new key store for pks built and proved beside the live one (hs_committee_stage_register), switched in by committee_commit:
  // stage + commit leaves the engine as hs_committee_register(pks) at the returned window.  key_bits 0: the widest window that fits beside
  // the live store; 8..17: that window.  Returns ceil(N / 32) words of key validity and the window.  Throws EngineError on any failure
  // (the live committee is untouched).
  std::pair<std::vector<uint32_t>, int> committee_stage_register(const uint8_t *pks, size_t N, int key_bits = 0) const {
    std::vector<uint32_t> valid((N + 31) / 32);
    int bits = 0;
    check(hs_committee_stage_register(ctx_, pks, N, key_bits, valid.data(), &bits), "hs_committee_stage_register");
    return {valid, bits};
  }
  std::string error() const { return hs_last_error(ctx_); }

 private:
  hs_ctx *ctx_ = nullptr;
  bool owned_ = true;
};

// RAII handle on hs_multi_* (hs_crypto.h): several member contexts in this process.  A verify call of at least HS_MULTI_MIN_SHARD records
// per member is sharded across the members, a smaller one runs whole on one member (round-robin); verdicts equal the same Engine call
// bit for bit.  Outputs are bitmaps as in the C ABI: bit (i & 31) of word (i >> 5).  Destroy every VerifyQueue made on a member first.
class MultiEngine {
 public:
  explicit MultiEngine(const std::vector<int> &devices, uint32_t flags = 0) {
    if (hs_multi_create(&m_, devices.data(), devices.size(), flags) != HS_OK)
      throw EngineError("hs_multi_create failed (no GPU, bad ordinal?) — there is no CPU fallback");
    for (size_t i = 0; i < devices.size(); i++) members_.emplace_back(new Engine(hs_multi_member(m_, i), Engine::Borrowed{}));
  }
  ~MultiEngine() {
    members_.clear();
    hs_multi_destroy(m_);
  }
  MultiEngine(const MultiEngine &) = delete;
  MultiEngine &operator=(const MultiEngine &) = delete;
  hs_multi *raw() const { return m_; }
  size_t size() const { return members_.size(); }
  // Member i: every single-device call works on it (a VerifyQueue, say).  Do not change its committee directly.
  const Engine &member(size_t i) const { return *members_.at(i); }
  void check(int rc, const char *what) const {
    if (rc != HS_OK) throw EngineError(std::string(what) + ": " + hs_multi_last_error(m_));
  }
  std::string error() const { return hs_multi_last_error(m_); }
  // The same committee on every member; returns ceil(N / 32) words of key validity.
  std::vector<uint32_t> register_committee(const uint8_t *pks, size_t N) {
    std::vector<uint32_t> valid((N + 31) / 32);
    check(hs_multi_committee_register(m_, pks, N, valid.data()), "hs_multi_committee_register");
    return valid;
  }
  // Returns the indices of the added keys, the same on every member.
  std::vector<uint32_t> update_committee(const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove) {
    std::vector<uint32_t> idx(n_add);
    check(hs_multi_committee_update(m_, add_pks, n_add, remove_idx, n_remove, idx.data()), "hs_multi_committee_update");
    return idx;
  }
  // The staged committee change on every member, member by member through the single-context calls (as a repair is): stages on every
  // member at once, one thread each, and returns the indices, the same on every member.  If any member fails, or the members return
  // different indices, the stage is discarded on every member and EngineError thrown: nothing stays staged.
  std::vector<uint32_t> stage_committee(const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove) {
    std::vector<std::future<std::vector<uint32_t>>> parts;
    for (auto &e : members_)
      parts.push_back(std::async(std::launch::async, [&e, add_pks, n_add, remove_idx, n_remove] {
        return e->committee_stage(add_pks, n_add, remove_idx, n_remove);
      }));
    std::vector<std::vector<uint32_t>> idx;
    std::string err;
    for (auto &p : parts) {
      try {
        idx.push_back(p.get());
      } catch (const EngineError &x) {
        if (err.empty()) err = x.what();
      }
    }
    for (size_t i = 1; err.empty() && i < idx.size(); i++)
      if (idx[i] != idx[0]) err = "stage_committee: member " + std::to_string(i) + " gave other indices than member 0";
    if (!err.empty()) {
      for (auto &e : members_) hs_committee_discard(e->raw());
      throw EngineError(err);
    }
    return idx.at(0);
  }
  // The staged registration on every member, member by member through the single-context call: stages on every member at once, one
  // thread each, and returns the validity words and the window, the same on every member.  If any member fails, or the members differ
  // in either, the stage is discarded on every member and EngineError thrown: every member keeps its committee.  commit_committee
  // switches it in.
  std::pair<std::vector<uint32_t>, int> stage_register_committee(const uint8_t *pks, size_t N, int key_bits = 0) {
    std::vector<std::future<std::pair<std::vector<uint32_t>, int>>> parts;
    for (auto &e : members_)
      parts.push_back(std::async(std::launch::async, [&e, pks, N, key_bits] { return e->committee_stage_register(pks, N, key_bits); }));
    std::vector<std::pair<std::vector<uint32_t>, int>> res;
    std::string err;
    for (auto &p : parts) {
      try {
        res.push_back(p.get());
      } catch (const EngineError &x) {
        if (err.empty()) err = x.what();
      }
    }
    for (size_t i = 1; err.empty() && i < res.size(); i++)
      if (res[i] != res[0]) err = "stage_register_committee: member " + std::to_string(i) + " gave other validity or window than member 0";
    if (!err.empty()) {
      for (auto &e : members_) hs_committee_discard(e->raw());
      throw EngineError(err);
    }
    return res.at(0);
  }
  // hs_committee_commit on every member.  After a failure the members may differ: re-register.
  void commit_committee() {
    for (auto &e : members_) e->committee_commit();
  }
  void discard_committee() {
    for (auto &e : members_) e->committee_discard();
  }
  std::vector<uint32_t> verify_rec128(const hs_rec128 *recs, size_t n, uint32_t mode = HS_MODE_STRICT) {
    std::vector<uint32_t> bm((n + 31) / 32);
    check(hs_multi_verify_rec128(m_, recs, n, mode, bm.data()), "hs_multi_verify_rec128");
    return bm;
  }
  // key_i = pk[i] (pk != nullptr) or committee key validator_idx[i].
  std::vector<uint32_t> verify_msgs(const uint8_t *sig, const uint8_t *pk, const uint32_t *validator_idx, const uint8_t *msgs, size_t msg_len, size_t n,
                                    uint32_t mode = HS_MODE_STRICT) {
    std::vector<uint32_t> bm((n + 31) / 32);
    check(hs_multi_verify_msgs(m_, sig, pk, validator_idx, msgs, msg_len, n, mode, bm.data()), "hs_multi_verify_msgs");
    return bm;
  }
  // Group words; item words go to out_item_bitmap when it is not null.
  std::vector<uint32_t> verify_groups(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                                      const uint32_t *validator_idx, const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *modes,
                                      size_t n_items, size_t n_groups, uint32_t *out_item_bitmap = nullptr) {
    std::vector<uint32_t> groups((n_groups + 31) / 32);
    check(hs_multi_verify_groups(m_, preimages, pre_off, n_msgs, sig, pk, validator_idx, msg_idx, group_idx, modes, n_items, n_groups, out_item_bitmap,
                                 groups.data()),
          "hs_multi_verify_groups");
    return groups;
  }

 private:
  hs_multi *m_ = nullptr;
  std::vector<std::unique_ptr<Engine>> members_;
};

// The verify queue's ring has no room for the request right now (HS_ERR_NOMEM): back-pressure, retry once requests complete.
struct QueueFull : EngineError {
  QueueFull() : EngineError("hs_queue_submit: the verify queue's ring is full") {}
};

// Verdicts of a batch request (VerifyQueue::submit_batch): one per group, one per item.
struct BatchVerdicts {
  std::vector<bool> groups, items;
};

// RAII handle on hs_queue_* (hs_crypto.h): many tasks submit small verifies (a Vote, a Timeout / Block author, a small QC) at
// once and share latency-path launches.  Each future yields the request's verdicts, bit-identical to hs_verify_rec128, or throws
// EngineError on an engine failure (reject every signature).  Destruction completes every request in flight.
class VerifyQueue {
 public:
  explicit VerifyQueue(const Engine &e, size_t ring_records = 0) : e_(e) { e.check(hs_queue_create(e.raw(), ring_records, &q_), "hs_queue_create"); }
  ~VerifyQueue() { hs_queue_destroy(q_); }
  VerifyQueue(const VerifyQueue &) = delete;
  VerifyQueue &operator=(const VerifyQueue &) = delete;

  // 1..64 records, HS_MODE_*.  Throws QueueFull when the ring is full, EngineError on a bad argument.
  std::future<std::vector<bool>> submit(const hs_rec128 *recs, size_t n, uint32_t mode = HS_MODE_STRICT) {
    auto *p = new Pending{std::promise<std::vector<bool>>(), n};
    std::future<std::vector<bool>> f = p->promise.get_future();
    const int rc = hs_queue_submit(q_, recs, n, mode, &VerifyQueue::done, p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit");
    }
    return f;
  }

  // One consensus message's whole certificate as ONE request (hs_queue_submit_group): a Block (author strict + QC votes batch-eq
  // + TC votes strict), a Timeout with its high_qc, a TC, a QC.  n = 1 .. ring capacity, modes[i] = HS_MODE_* of record i
  // (nullptr = all strict).  Throws QueueFull when the ring has no room now (verify synchronously), EngineError on a bad argument.
  std::future<std::vector<bool>> submit_group(const hs_rec128 *recs, size_t n, const uint8_t *modes = nullptr) {
    auto *p = new Pending{std::promise<std::vector<bool>>(), n};
    std::future<std::vector<bool>> f = p->promise.get_future();
    const int rc = hs_queue_submit_group(q_, recs, n, modes, &VerifyQueue::done, p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit_group");
    }
    return f;
  }

  // The same with the signed preimages instead of their Digests (hs_queue_submit_msgs): record i is (sig[i], pk[i]) over
  // Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1])), hashed on the GPU — the arrays hs_ingest_consensus_frames
  // writes for one frame.  Throws QueueFull when the ring or the preimage arena has no room now, EngineError on a bad argument.
  std::future<std::vector<bool>> submit_msgs(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                                             const uint32_t *msg_idx, size_t n, const uint8_t *modes = nullptr) {
    auto *p = new Pending{std::promise<std::vector<bool>>(), n};
    std::future<std::vector<bool>> f = p->promise.get_future();
    const int rc = hs_queue_submit_msgs(q_, preimages, pre_off, n_msgs, sig, pk, msg_idx, modes, n, &VerifyQueue::done, p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit_msgs");
    }
    return f;
  }

  // Counters since creation (hs_queue_stats): [0] k_verify_small launches, [1] their records, [2] k_verify_bulk launches,
  // [3] their records, [4] slow-path requests, [5] their records.
  std::array<uint64_t, HS_QUEUE_STATS> stats() const {
    std::array<uint64_t, HS_QUEUE_STATS> s{};
    e_.check(hs_queue_stats(q_, s.data()), "hs_queue_stats");
    return s;
  }
  // hs_queue_digest_stats: [0] k_queue_digests launches, [1] preimages hashed, [2] their bytes, [3] submit_msgs requests.
  std::array<uint64_t, HS_QUEUE_DIGEST_STATS> digest_stats() const {
    std::array<uint64_t, HS_QUEUE_DIGEST_STATS> s{};
    e_.check(hs_queue_digest_stats(q_, s.data()), "hs_queue_digest_stats");
    return s;
  }
  // hs_queue_cert_cache: keep up to max_bytes of verified certificates (0 = off, the default).  Verdicts do not change.
  void cert_cache(size_t max_bytes) { e_.check(hs_queue_cert_cache(q_, max_bytes), "hs_queue_cert_cache"); }
  // hs_queue_cert_stats: [0] spans looked up, [1] hits, [2] in-flight joins, [3] records answered without verifying them,
  // [4] spans inserted, [5] bytes held now.
  std::array<uint64_t, HS_QUEUE_CERT_STATS> cert_stats() const {
    std::array<uint64_t, HS_QUEUE_CERT_STATS> s{};
    e_.check(hs_queue_cert_stats(q_, s.data()), "hs_queue_cert_stats");
    return s;
  }
  // hs_queue_sig_cache: a table of at least `entries` accepted records (0 = off, the default).  Verdicts do not change.
  void sig_cache(size_t entries) { e_.check(hs_queue_sig_cache(q_, entries), "hs_queue_sig_cache"); }
  // hs_queue_sig_stats: [0] records probed, [1] hits, [2] inserts, [3] inserts that evicted a live entry, [4] entries held now.
  std::array<uint64_t, HS_QUEUE_SIG_STATS> sig_stats() const {
    std::array<uint64_t, HS_QUEUE_SIG_STATS> s{};
    e_.check(hs_queue_sig_stats(q_, s.data()), "hs_queue_sig_stats");
    return s;
  }
  // hs_queue_sig_share: the synchronous verify calls on the context and the batch lane probe and fill this queue's signature cache
  // (off by default; needs the cache on, one queue per context).  Verdicts do not change.
  void sig_share(bool on) { e_.check(hs_queue_sig_share(q_, on ? 1 : 0), "hs_queue_sig_share"); }
  // hs_queue_sig_share_stats: [0] records probed, [1] hits, [2] inserts, [3] inserts that evicted a live entry, [4] shared passes.
  std::array<uint64_t, HS_QUEUE_SIG_SHARE_STATS> sig_share_stats() const {
    std::array<uint64_t, HS_QUEUE_SIG_SHARE_STATS> s{};
    e_.check(hs_queue_sig_share_stats(q_, s.data()), "hs_queue_sig_share_stats");
    return s;
  }
  // hs_queue_sig_audit: re-checks every held entry of buckets [first_bucket, first_bucket + n_buckets) (0: to the end) from its bytes and
  // corrects the flag bytes that disagree.  [0] held, [1] corrected, [2] skipped, [3] first corrected position (UINT64_MAX: none),
  // [4] its stored flags, [5] its derived flags, [6] its HS_WHY_* mask.  Throws EngineError when the cache is off or the range leaves it.
  std::array<uint64_t, HS_QUEUE_SIG_AUDIT_OUT> sig_audit(size_t first_bucket = 0, size_t n_buckets = 0) {
    std::array<uint64_t, HS_QUEUE_SIG_AUDIT_OUT> s{};
    e_.check(hs_queue_sig_audit(q_, first_bucket, n_buckets, s.data()), "hs_queue_sig_audit");
    return s;
  }
  // hs_queue_sig_audit_stats: [0] audits, [1] entries re-checked, [2] corrected, [3] skipped, [4] full passes of the table.
  std::array<uint64_t, HS_QUEUE_SIG_AUDIT_STATS> sig_audit_stats() const {
    std::array<uint64_t, HS_QUEUE_SIG_AUDIT_STATS> s{};
    e_.check(hs_queue_sig_audit_stats(q_, s.data()), "hs_queue_sig_audit_stats");
    return s;
  }
  hs_queue *raw() const { return q_; }
  // hs_queue_generic: verify requests with keys outside the committee on the GPU, not on the dispatcher thread (off by default;
  // off drains the generic launches in flight).  Verdicts do not change.
  void generic(bool on) { e_.check(hs_queue_generic(q_, on ? 1 : 0), "hs_queue_generic"); }
  // hs_queue_generic_stats: [0] k_queue_generic launches, [1] records they carried, [2] requests.
  std::array<uint64_t, HS_QUEUE_GENERIC_STATS> generic_stats() const {
    std::array<uint64_t, HS_QUEUE_GENERIC_STATS> s{};
    e_.check(hs_queue_generic_stats(q_, s.data()), "hs_queue_generic_stats");
    return s;
  }
  // hs_queue_batch: turn the batch lane on for requests of up to max_items items and max_bytes of arena region (0, 0 = off, the
  // default).  Resizing or turning it off first waits for the batch requests already submitted.
  void batch(size_t max_items, size_t max_bytes) { e_.check(hs_queue_batch(q_, max_items, max_bytes), "hs_queue_batch"); }
  // hs_verify_groups with key bytes as ONE non-blocking request on the batch lane (hs_queue_submit_batch).  The future yields the
  // group and item verdicts, bit for bit those of hs_verify_groups, or throws EngineError on an engine failure (reject every
  // group).  Throws QueueFull when the lane's arena has no room now, EngineError on a bad argument or when the lane is off.
  std::future<BatchVerdicts> submit_batch(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                                          const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *modes, size_t n_items, size_t n_groups) {
    auto *p = new BatchPending{std::promise<BatchVerdicts>(), n_items, n_groups};
    std::future<BatchVerdicts> f = p->promise.get_future();
    const int rc = hs_queue_submit_batch(q_, preimages, pre_off, n_msgs, sig, pk, msg_idx, group_idx, modes, n_items, n_groups, &VerifyQueue::batch_done,
                                         p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit_batch");
    }
    return f;
  }
  // hs_queue_batch_stats: [0] batch passes, [1] items, [2] groups, [3] preimage bytes hashed, [4] items outside the committee.
  std::array<uint64_t, HS_QUEUE_BATCH_STATS> batch_stats() const {
    std::array<uint64_t, HS_QUEUE_BATCH_STATS> s{};
    e_.check(hs_queue_batch_stats(q_, s.data()), "hs_queue_batch_stats");
    return s;
  }
  // hs_queue_explain: turn the explain lane on for requests of up to max_records records and max_bytes of arena region (0, 0 = off,
  // the default).  Resizing or turning it off first waits for the explain requests already submitted.
  void explain(size_t max_records, size_t max_bytes) { e_.check(hs_queue_explain(q_, max_records, max_bytes), "hs_queue_explain"); }
  // Engine::explain as ONE non-blocking request on the explain lane (hs_queue_submit_explain).  The future yields one HS_WHY_* byte per
  // record, byte for byte those of hs_explain_rec128, or throws EngineError on an engine failure (explain nothing).  Throws QueueFull
  // when the lane's arena has no room now, EngineError on a bad argument or when the lane is off.
  std::future<std::vector<uint8_t>> submit_explain(const hs_rec128 *recs, size_t n) {
    auto *p = new WhyPending{std::promise<std::vector<uint8_t>>(), n};
    std::future<std::vector<uint8_t>> f = p->promise.get_future();
    const int rc = hs_queue_submit_explain(q_, recs, n, &VerifyQueue::why_done, p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit_explain");
    }
    return f;
  }
  // The same with the signed preimages instead of their Digests (hs_queue_submit_explain_msgs): the arrays of submit_msgs without modes.
  std::future<std::vector<uint8_t>> submit_explain_msgs(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig,
                                                        const uint8_t *pk, const uint32_t *msg_idx, size_t n) {
    auto *p = new WhyPending{std::promise<std::vector<uint8_t>>(), n};
    std::future<std::vector<uint8_t>> f = p->promise.get_future();
    const int rc = hs_queue_submit_explain_msgs(q_, preimages, pre_off, n_msgs, sig, pk, msg_idx, n, &VerifyQueue::why_done, p, nullptr);
    if (rc != HS_OK) {
      delete p;
      if (rc == HS_ERR_NOMEM) throw QueueFull();
      e_.check(rc, "hs_queue_submit_explain_msgs");
    }
    return f;
  }
  // hs_queue_explain_stats: [0] k_queue_explain launches, [1] records they carried, [2] requests.
  std::array<uint64_t, HS_QUEUE_EXPLAIN_STATS> explain_stats() const {
    std::array<uint64_t, HS_QUEUE_EXPLAIN_STATS> s{};
    e_.check(hs_queue_explain_stats(q_, s.data()), "hs_queue_explain_stats");
    return s;
  }

 private:
  struct WhyPending {
    std::promise<std::vector<uint8_t>> promise;
    size_t n;
  };
  // runs once per explain request on the queue's thread: the words hold the why bytes, byte i of the little-endian packing = record i
  static void why_done(void *user, size_t, int status, const uint32_t *bitmap) {
    WhyPending *p = static_cast<WhyPending *>(user);
    if (status == HS_OK) {
      std::vector<uint8_t> v(p->n);
      for (size_t i = 0; i < p->n; i++) v[i] = (uint8_t)(bitmap[i >> 2] >> (8 * (i & 3)));
      p->promise.set_value(std::move(v));
    } else {
      p->promise.set_exception(std::make_exception_ptr(EngineError("verify queue explain: engine failure (status " + std::to_string(status) + ")")));
    }
    delete p;
  }
  struct BatchPending {
    std::promise<BatchVerdicts> promise;
    size_t n_items, n_groups;
  };
  // runs once per batch request on the queue's thread: the bitmap holds the group words, then the item words
  static void batch_done(void *user, size_t, int status, const uint32_t *bitmap) {
    BatchPending *p = static_cast<BatchPending *>(user);
    if (status == HS_OK) {
      BatchVerdicts v{std::vector<bool>(p->n_groups), std::vector<bool>(p->n_items)};
      const uint32_t *items = bitmap + (p->n_groups + 31) / 32;
      for (size_t j = 0; j < p->n_groups; j++) v.groups[j] = (bitmap[j >> 5] >> (j & 31)) & 1u;
      for (size_t i = 0; i < p->n_items; i++) v.items[i] = (items[i >> 5] >> (i & 31)) & 1u;
      p->promise.set_value(std::move(v));
    } else {
      p->promise.set_exception(std::make_exception_ptr(EngineError("verify queue batch: engine failure (status " + std::to_string(status) + ")")));
    }
    delete p;
  }
  struct Pending {
    std::promise<std::vector<bool>> promise;
    size_t n;
  };
  // runs once per request on the queue's thread
  static void done(void *user, size_t, int status, const uint32_t *bitmap) {
    Pending *p = static_cast<Pending *>(user);
    if (status == HS_OK) {
      std::vector<bool> v(p->n);
      for (size_t i = 0; i < p->n; i++) v[i] = (bitmap[i >> 5] >> (i & 31)) & 1u;
      p->promise.set_value(std::move(v));
    } else {
      p->promise.set_exception(std::make_exception_ptr(EngineError("verify queue: engine failure (status " + std::to_string(status) + ")")));
    }
    delete p;
  }
  const Engine &e_;
  hs_queue *q_ = nullptr;
};

inline void Engine::scrub_sig_cache(const VerifyQueue *q, uint32_t buckets_per_tick) const {
  check(hs_scrub_sig_cache(ctx_, q ? q->raw() : nullptr, buckets_per_tick), "hs_scrub_sig_cache");
}

struct Digest {  // crypto/src/lib.rs:22
  std::array<uint8_t, 32> bytes{};
  size_t size() const { return 32; }
  std::vector<uint8_t> to_vec() const { return {bytes.begin(), bytes.end()}; }
  bool operator==(const Digest &o) const { return bytes == o.bytes; }
  // Digest(SHA-512(data)[..32]) — the Hash impls of consensus/src/messages.rs and mempool/src/processor.rs:30
  static Digest of(const Engine &e, const uint8_t *data, size_t len) {
    Digest d;
    const uint64_t off[2] = {0, (uint64_t)len};
    e.check(hs_digest32_batch(e.raw(), data, off, 1, d.bytes.data()), "hs_digest32_batch");
    return d;
  }
};

struct PublicKey {  // crypto/src/lib.rs:66
  std::array<uint8_t, 32> bytes{};
  bool operator==(const PublicKey &o) const { return bytes == o.bytes; }
};

struct Signature {  // crypto/src/lib.rs:179-182; default = 64 zero bytes (the "invalid" signature of crypto_tests.rs:111)
  std::array<uint8_t, 32> part1{}, part2{};
  static Signature from_bytes(const uint8_t b[64]) {
    Signature s;
    std::memcpy(s.part1.data(), b, 32);
    std::memcpy(s.part2.data(), b + 32, 32);
    return s;
  }
  std::array<uint8_t, 64> flatten() const {  // lib.rs:193-198
    std::array<uint8_t, 64> f;
    std::memcpy(f.data(), part1.data(), 32);
    std::memcpy(f.data() + 32, part2.data(), 32);
    return f;
  }
  // Signature::verify (lib.rs:200-204): dalek verify_strict.  Throws CryptoError on Err.
  void verify(const Engine &e, const Digest &digest, const PublicKey &public_key) const {
    hs_rec128 rec;
    const auto f = flatten();
    std::memcpy(rec.sig, f.data(), 64);
    std::memcpy(rec.pk, public_key.bytes.data(), 32);
    std::memcpy(rec.msg, digest.bytes.data(), 32);
    uint32_t word = 0;
    e.check(hs_verify_strict_batch(e.raw(), &rec, 1, &word), "hs_verify_strict_batch");
    if (!(word & 1u)) throw CryptoError();
  }
  // Signature::verify_batch (lib.rs:206-219): one digest, votes = (PublicKey, Signature) pairs.
  static void verify_batch(const Engine &e, const Digest &digest, const std::vector<std::pair<PublicKey, Signature>> &votes) {
    std::vector<hs_vote> v(votes.size());
    for (size_t i = 0; i < votes.size(); i++) {
      std::memcpy(v[i].pk, votes[i].first.bytes.data(), 32);
      const auto f = votes[i].second.flatten();
      std::memcpy(v[i].sig, f.data(), 64);
    }
    int ok = 0;
    e.check(hs_verify_batch_shared_msg(e.raw(), digest.bytes.data(), v.data(), v.size(), &ok, nullptr), "hs_verify_batch_shared_msg");
    if (!ok) throw CryptoError();
  }
};

}  // namespace hs
