// Multi-device context (include/hs_crypto.h, "several GPUs in one process"): N ordinary contexts, its members, and the host code that
// splits one host-pointer verify call across them.  Only the members' public entry points are called here, so every kernel that runs
// is a member's, under that member's own mutex.
//   - A call of at least HS_MULTI_MIN_SHARD records per member is sharded: member i verifies a contiguous record range, every range
//     but the last starts at a multiple of 32 records, so each member writes whole words of the caller's bitmap and no word is shared.
//     Sharded calls hold the multi-context's mutex; worker k runs member k's range, the calling thread member 0's.
//   - A smaller call runs whole on one member, picked round-robin without the multi-context's mutex, so small calls from several
//     threads run on different GPUs at once.
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <new>
#include <string>
#include <system_error>
#include <thread>
#include <vector>

#include "../../include/hs_crypto.h"
#include "hs_args.h"

struct hs_multi {
  std::vector<hs_ctx *> members;
  std::vector<int> devices;          // CUDA ordinal of each member
  std::vector<std::thread> workers;  // workers[k - 1] runs member k's part of every fan-out
  std::mutex mu;                     // serialises fan-outs: sharded calls and committee changes
  std::atomic<uint64_t> next{0};     // round-robin counter of the calls that run whole on one member
  // the fan-out in progress (guarded by job_mu)
  std::mutex job_mu;
  std::condition_variable job_cv, done_cv;
  const std::function<int(size_t)> *job = nullptr;
  uint64_t job_seq = 0;
  size_t pending = 0;
  std::vector<int> rc;
  bool stop = false;
  std::mutex err_mu;
  std::string err = "ok";
};

static int mfail(hs_multi *m, int code, const std::string &what) {
  if (m) {
    std::lock_guard<std::mutex> g(m->err_mu);
    m->err = what;
  }
  return code;
}
// A member's failure: its status, and hs_multi_last_error names the member and gives its hs_last_error.
static int member_fail(hs_multi *m, const char *entry, size_t i, int code) {
  return mfail(m, code, std::string(entry) + ": member " + std::to_string(i) + " (device " + std::to_string(m->devices[i]) + "): " +
                            hs_last_error(m->members[i]));
}

static void worker_main(hs_multi *m, size_t k) {
  uint64_t seen = 0;
  std::unique_lock<std::mutex> lk(m->job_mu);
  for (;;) {
    m->job_cv.wait(lk, [&] { return m->stop || m->job_seq != seen; });
    if (m->stop) return;
    seen = m->job_seq;
    const std::function<int(size_t)> *job = m->job;
    lk.unlock();
    const int rc = (*job)(k);
    lk.lock();
    m->rc[k] = rc;
    if (--m->pending == 0) m->done_cv.notify_all();
  }
}
// Runs fn(i) for every member i at once (member 0 on the calling thread, which holds m->mu) and returns the first failing member's
// status, its index in *failed.
static int fan_out(hs_multi *m, const std::function<int(size_t)> &fn, size_t *failed) {
  const size_t n = m->members.size();
  {
    std::lock_guard<std::mutex> g(m->job_mu);
    m->rc.assign(n, HS_OK);
    m->job = &fn;
    m->pending = n - 1;
    m->job_seq++;
  }
  m->job_cv.notify_all();
  const int rc0 = fn(0);
  std::unique_lock<std::mutex> lk(m->job_mu);
  m->done_cv.wait(lk, [&] { return m->pending == 0; });
  m->rc[0] = rc0;
  m->job = nullptr;
  for (size_t i = 0; i < n; i++)
    if (m->rc[i] != HS_OK) {
      *failed = i;
      return m->rc[i];
    }
  return HS_OK;
}

// Record range [lo, hi) of member i out of k over n records, as hotstuff_b200.sharding.shard_range: every range but the last holds
// ceil(n / k) rounded up to 32 records.
struct shard {
  size_t lo, hi;
};
static shard shard_of(size_t n, size_t i, size_t k) {
  const size_t per = ((n + k - 1) / k + 31) & ~(size_t)31;
  const size_t lo = i * per < n ? i * per : n;
  return {lo, lo + per < n ? lo + per : n};
}
static bool sharded(const hs_multi *m, size_t n) { return m->members.size() > 1 && n / m->members.size() >= HS_MULTI_MIN_SHARD; }
// The member that runs a call whole.
static size_t pick(hs_multi *m) { return (size_t)(m->next.fetch_add(1, std::memory_order_relaxed) % m->members.size()); }

// A call that runs whole on one member, or sharded across all of them: run(i, range) is member i's part.
template <class Run>
static int dispatch(hs_multi *m, const char *entry, size_t n, Run run) {
  if (!sharded(m, n)) {
    const size_t i = pick(m);
    const int rc = run(i, shard{0, n});
    return rc == HS_OK ? HS_OK : member_fail(m, entry, i, rc);
  }
  std::lock_guard<std::mutex> g(m->mu);
  const size_t k = m->members.size();
  size_t failed = 0;
  const int rc = fan_out(m, [&](size_t i) {
    const shard s = shard_of(n, i, k);
    return s.hi > s.lo ? run(i, s) : HS_OK;
  }, &failed);
  return rc == HS_OK ? HS_OK : member_fail(m, entry, failed, rc);
}

extern "C" {

int hs_multi_create(hs_multi **out, const int *devices, size_t n_devices, uint32_t flags) {
  if (!out) return HS_ERR_ARG;
  *out = nullptr;
  if (!devices || n_devices == 0) return HS_ERR_ARG;
  hs_multi *m = new (std::nothrow) hs_multi();
  if (!m) return HS_ERR_NOMEM;
  int rc = HS_OK;
  for (size_t i = 0; i < n_devices && rc == HS_OK; i++) {
    hs_ctx *c = nullptr;
    rc = hs_ctx_create(&c, devices[i], flags);
    if (rc == HS_OK) {
      m->members.push_back(c);
      m->devices.push_back(devices[i]);
    }
  }
  if (rc == HS_OK) {
    try {
      for (size_t k = 1; k < n_devices; k++) m->workers.emplace_back(worker_main, m, k);
    } catch (const std::system_error &) {
      rc = HS_ERR_NOMEM;
    }
  }
  if (rc != HS_OK) {
    hs_multi_destroy(m);
    return rc;
  }
  *out = m;
  return HS_OK;
}

void hs_multi_destroy(hs_multi *m) {
  if (!m) return;
  {
    std::lock_guard<std::mutex> g(m->job_mu);
    m->stop = true;
  }
  m->job_cv.notify_all();
  for (std::thread &t : m->workers) t.join();
  for (hs_ctx *c : m->members) hs_ctx_destroy(c);  // destroys the verify queues created on the members too
  delete m;
}

const char *hs_multi_last_error(const hs_multi *m) { return m ? m->err.c_str() : "null context"; }
size_t hs_multi_members(const hs_multi *m) { return m ? m->members.size() : 0; }
hs_ctx *hs_multi_member(hs_multi *m, size_t i) { return (m && i < m->members.size()) ? m->members[i] : nullptr; }

int hs_multi_committee_register(hs_multi *m, const uint8_t *pks, size_t N, uint32_t *out_valid_bitmap) {
  if (!m || (N && !pks)) return mfail(m, HS_ERR_ARG, "hs_multi_committee_register: bad argument");
  std::lock_guard<std::mutex> g(m->mu);
  const size_t k = m->members.size(), words = (N + 31) / 32;
  std::vector<std::vector<uint32_t>> valid(k, std::vector<uint32_t>(words));
  size_t failed = 0;
  int rc = fan_out(m, [&](size_t i) { return hs_committee_register(m->members[i], pks, N, valid[i].data()); }, &failed);
  if (rc != HS_OK) member_fail(m, "hs_multi_committee_register", failed, rc);
  for (size_t i = 1; i < k && rc == HS_OK; i++)
    if (valid[i] != valid[0])
      rc = mfail(m, HS_ERR_CUDA, "hs_multi_committee_register: member " + std::to_string(i) + " found other keys valid than member 0");
  if (rc != HS_OK) {  // a failed registration leaves NO committee, on any member
    fan_out(m, [&](size_t i) { return hs_committee_register(m->members[i], nullptr, 0, nullptr); }, &failed);
    return rc;
  }
  if (out_valid_bitmap) std::copy(valid[0].begin(), valid[0].end(), out_valid_bitmap);
  return HS_OK;
}

int hs_multi_committee_update(hs_multi *m, const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove,
                              uint32_t *out_add_idx) {
  if (!m) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(m->mu);
  const size_t k = m->members.size();
  std::vector<std::vector<uint32_t>> idx(k, std::vector<uint32_t>(n_add));
  size_t failed = 0;
  const int rc = fan_out(m, [&](size_t i) {
    return hs_committee_update(m->members[i], add_pks, n_add, remove_idx, n_remove, out_add_idx ? idx[i].data() : nullptr);
  }, &failed);
  if (rc != HS_OK) return member_fail(m, "hs_multi_committee_update", failed, rc);
  for (size_t i = 1; i < k; i++)
    if (idx[i] != idx[0])
      return mfail(m, HS_ERR_CUDA, "hs_multi_committee_update: member " + std::to_string(i) + " gave other indices than member 0 (re-register)");
  if (out_add_idx) std::copy(idx[0].begin(), idx[0].end(), out_add_idx);
  return HS_OK;
}

int hs_multi_verify_rec128(hs_multi *m, const hs_rec128 *recs, size_t n, uint32_t mode, uint32_t *out_bitmap) {
  if (!m) return HS_ERR_ARG;
  if (const char *why = hs_args::rec128(recs, n, mode, out_bitmap)) return mfail(m, HS_ERR_ARG, std::string("hs_multi_verify_rec128: ") + why);
  if (n == 0) return HS_OK;
  return dispatch(m, "hs_multi_verify_rec128", n, [&](size_t i, shard s) {
    return hs_verify_rec128(m->members[i], recs + s.lo, s.hi - s.lo, mode, out_bitmap + s.lo / 32);
  });
}

int hs_multi_verify_msgs(hs_multi *m, const uint8_t *sig, const uint8_t *pk, const uint32_t *vidx, const uint8_t *msgs, size_t msg_len, size_t n,
                         uint32_t mode, uint32_t *out_bitmap) {
  if (!m) return HS_ERR_ARG;
  if (const char *why = hs_args::msgs(sig, pk, vidx, msgs, msg_len, n, mode, out_bitmap))
    return mfail(m, HS_ERR_ARG, std::string("hs_multi_verify_msgs: ") + why);
  if (n == 0) return HS_OK;
  return dispatch(m, "hs_multi_verify_msgs", n, [&](size_t i, shard s) {
    return hs_verify_msgs(m->members[i], sig + 64 * s.lo, pk ? pk + 32 * s.lo : nullptr, vidx ? vidx + s.lo : nullptr, msgs + msg_len * s.lo, msg_len,
                          s.hi - s.lo, mode, out_bitmap + s.lo / 32);
  });
}

int hs_multi_verify_groups(hs_multi *m, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                           const uint32_t *vidx, const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *mode, size_t n_items,
                           size_t n_groups, uint32_t *out_item_bitmap, uint32_t *out_group_bitmap) {
  if (!m) return HS_ERR_ARG;
  if (const char *why = hs_args::groups(preimages, pre_off, n_msgs, sig, pk, vidx, msg_idx, group_idx, mode, n_items, n_groups, out_group_bitmap))
    return mfail(m, HS_ERR_ARG, std::string("hs_multi_verify_groups: ") + why);
  const char *entry = "hs_multi_verify_groups";
  const auto items = [&](size_t i, shard s, uint32_t *groups) {
    return hs_verify_groups(m->members[i], preimages, pre_off, n_msgs, sig + 64 * s.lo, pk ? pk + 32 * s.lo : nullptr, vidx ? vidx + s.lo : nullptr,
                            msg_idx + s.lo, group_idx + s.lo, mode ? mode + s.lo : nullptr, s.hi - s.lo, n_groups,
                            out_item_bitmap ? out_item_bitmap + s.lo / 32 : nullptr, groups);
  };
  if (!sharded(m, n_items)) return dispatch(m, entry, n_items, [&](size_t i, shard s) { return items(i, s, out_group_bitmap); });
  // Each member ANDs its own items into its own group words (a group with no item in its range stays 1); the caller's group words are
  // the AND of the members' words.
  const size_t g_words = (n_groups + 31) / 32;
  std::vector<std::vector<uint32_t>> groups(m->members.size(), std::vector<uint32_t>(g_words, ~0u));
  const int rc = dispatch(m, entry, n_items, [&](size_t i, shard s) { return items(i, s, groups[i].data()); });
  if (rc != HS_OK) return rc;
  for (size_t w = 0; w < g_words; w++) {
    uint32_t v = groups[0][w];
    for (size_t i = 1; i < groups.size(); i++) v &= groups[i][w];
    out_group_bitmap[w] = v;
  }
  return HS_OK;
}

}  // extern "C"
