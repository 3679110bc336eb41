// hs_engine.cu — sm_90a kernels + the C ABI of include/hs_crypto.h.
//
// Hot path of asonnino/hotstuff's crypto crate (crypto/src/lib.rs:200-219 + the SHA-512 Digest call sites) rebuilt for
// H100.  No CPU path: if CUDA fails the call returns an error and the caller must reject.
//
// Throughput pipeline of one verify call (any n):
//   k_key_lookup      pk bytes -> committee index through a device hash table; misses -> compacted list
//                     (skipped when the caller gives validator indices)
//   k_verify_main<C>  registered / learned keys: SHA-512(R||A||M) -> k mod l -> [k](-A) + [S]B by table gathers only
//                     (17 + 11 mixed additions for 4,096 keys; no doublings, no decompression) -> (X:Y:Z) + meta
//   k_verify_main<G>  records whose key has no table: decompress A, radix-16 window for [k](-A); runs over the
//                     compacted list on a high-priority side stream, beside the pass above
//   k_verify_finish   two-level Montgomery-batched inversion, affine compare with R's encoding, small-order rule,
//                     32 verdicts -> one bitmap word, stored locally or into every peer GPU's buffer (fused all-gather,
//                     epoch flags exchanged by the last block); optionally on the context's tail stream (deferred mode)
// Latency pipeline (n <= 64, every key has a table): k_verify_small — ONE launch, a warp per signature sums the table entries
//   with a shuffle tree while a second warp decompresses R; inputs / verdicts in mapped pinned memory.
// Verify queue: small requests share k_verify_small launches; a large certificate gets k_verify_bulk (a thread per signature
//   from the queue's ring, the block's Z's inverted together, verdicts written by the same launch).
// Digest: k_digest32_fixed (staged coalesced loads, constant padding schedule), k_digest32 (any length), k_digest32_long
//   (one warp per long message, schedules expanded across lanes).
// Front ends: QC / TC / Timeout / Block groups with on-GPU digests and per-certificate AND; load-generation keygen / signer.
#include <cuda_runtime.h>
#include <pthread.h>
#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <type_traits>
#include <initializer_list>
#include <list>
#include <memory>
#include <mutex>
#include <new>
#include <optional>
#include <random>
#include <string>
#include <string_view>
#include <system_error>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/hs_crypto.h"
#include "hs_args.h"
#include "hs_selftest_vectors.h"
#include "key_index.h"
#include "verify_core.cuh"
#include "explain_select.cuh"

#define HS_THREADS 128
#define HS_FINISH_GROUP 16  // signatures whose Z's share one inversion
#define HS_LEARN_MAX 8192u  // unknown keys examined per call
#define HS_LEARN_PER_CALL 1024u  // new tables built per call at most (bounds the latency a flood of one-off keys can add to one call)
#define HS_CACHE_RESET_MIN_CALLS 64u  // a full cache is cleared at most once per this many verify calls

// ------------------------------------------------------------------------------------------------ input layout
// One descriptor covers every caller-facing layout: packed hs_rec128 records, separate sig/pk arrays with
// variable-length messages, QC votes sharing one digest, committee-indexed votes.
struct in_layout {
  const uint8_t *sig;   // 64-byte signature of record i at sig + i * sig_stride
  size_t sig_stride;
  const uint8_t *pk;    // 32-byte key of record i at pk + i * pk_stride (nullptr when only indices are given)
  size_t pk_stride;
  const uint32_t *vidx; // committee index per record (caller-given or produced by k_key_lookup); nullptr = none
  const uint8_t *msg;   // message i: off ? msg + off[i] : msg + (midx ? midx[i] : i) * msg_stride
  size_t msg_stride;
  const uint32_t *midx;
  const uint64_t *off;
  uint64_t fixed_len;   // message length when off == nullptr
  int aos128;           // 1: sig/pk/msg are the fields of packed 128-byte records at `sig` (coalesced staged loads)
};

__device__ __forceinline__ void load32(uint32_t (&w)[8], const uint8_t *p) {
  const uint32_t *s = reinterpret_cast<const uint32_t *>(p);  // every 32-byte field is 4-byte aligned in all layouts
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = __ldg(s + i);
}
// 32 bytes held as two 16-byte vectors -> 8 words
__device__ __forceinline__ void unpack8(uint32_t (&w)[8], uint4 lo, uint4 hi) {
  w[0] = lo.x; w[1] = lo.y; w[2] = lo.z; w[3] = lo.w;
  w[4] = hi.x; w[5] = hi.y; w[6] = hi.z; w[7] = hi.w;
}
// A 32-byte Digest (the first 8 words of a SHA-512 output) as two 16-byte stores; dst is 16-byte aligned.
__device__ __forceinline__ void store_digest32(uint32_t *dst, const uint32_t *h) {
  uint4 *d = reinterpret_cast<uint4 *>(dst);
  d[0] = make_uint4(h[0], h[1], h[2], h[3]);
  d[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

// A warp loads 32 rows of 128 bytes (rows warp_first .. warp_first + 31 of n; row(r) is the 16-byte aligned address of row
// warp_first + r) with fully coalesced 16-byte accesses, parks them in shared memory under an XOR swizzle, and every lane then
// reads back its own row conflict-free.  Rows past n read as zeros.  Every lane of the warp must call it, with lane = threadIdx.x
// & 31.  row() runs on every lane for every r, in range or not, so it may hold a full-warp shuffle.  The caller synchronises (warp
// or block) before smem_warp is written again.
template <class I, class Row>
__device__ __forceinline__ void warp_stage_rows128(uint4 (&q)[8], I n, I warp_first, Row row, uint4 *smem_warp, int lane) {
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int c = j * 32 + lane;  // chunk index inside the warp's 4 KB
    const int rec = c >> 3, part = c & 7;
    const uint4 *src = row(rec);  // outside the branch below: a shuffle there would diverge
    uint4 v = make_uint4(0, 0, 0, 0);
    if (warp_first + rec < n) v = __ldg(src + part);
    smem_warp[rec * 8 + (part ^ (rec & 7))] = v;
  }
  __syncwarp();
#pragma unroll
  for (int part = 0; part < 8; part++) q[part] = smem_warp[lane * 8 + (part ^ (lane & 7))];
}
// packed hs_rec128 records: sig.R | sig.S | pk | msg
__device__ __forceinline__ void warp_load_rec128(uint32_t (&sig_r)[8], uint32_t (&sig_s)[8], uint32_t (&pk)[8], uint32_t (&msg)[8],
                                                 const uint8_t *__restrict__ recs, size_t n, size_t warp_first, uint4 *smem_warp) {
  uint4 q[8];
  warp_stage_rows128(q, n, warp_first, [&](int r) { return reinterpret_cast<const uint4 *>(recs + (warp_first + r) * 128); }, smem_warp,
                     threadIdx.x & 31);
  __syncwarp();  // k_verify_main takes a block barrier next anyway; without this one its code schedules differently
  unpack8(sig_r, q[0], q[1]);
  unpack8(sig_s, q[2], q[3]);
  unpack8(pk, q[4], q[5]);
  unpack8(msg, q[6], q[7]);
}

// ------------------------------------------------------------------------------------------------ committee key lookup
// Open-addressing hash table over the registered keys: slot -> key index (HS_NO_KEY = empty).  Built on the host by key_index
// (key_index.h), probed here by one thread per record.
struct key_table {
  const uint32_t *slots;
  uint32_t mask;  // capacity - 1 (power of two)
  const uint8_t *pks;
  uint32_t n_keys;
};
// The key index the table maps key bytes k to (HS_NO_KEY: none) and, when found, the hash slot holding it.  BOUNDED (hs_table_audit,
// which must not trust the table it checks): an index at or past T.n_keys is a non-match instead of an address.
template <bool BOUNDED>
__device__ __forceinline__ uint32_t key_probe(const key_table &T, const uint32_t (&k)[8], uint32_t &pos) {
  uint32_t h = key_hash(k) & T.mask;
  for (uint32_t probe = 0; probe <= T.mask; probe++) {
    uint32_t idx = __ldg(T.slots + h);
    if (idx == HS_NO_KEY) break;
    if (!BOUNDED || idx < T.n_keys) {
      const uint32_t *cand = reinterpret_cast<const uint32_t *>(T.pks + (size_t)idx * 32);
      uint32_t diff = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) diff |= __ldg(cand + j) ^ k[j];
      if (diff == 0) {
        pos = h;
        return idx;
      }
    }
    h = (h + 1) & T.mask;
  }
  return HS_NO_KEY;
}
__global__ void __launch_bounds__(256) k_key_lookup(in_layout L, size_t n, key_table T, uint32_t *__restrict__ out_vidx,
                                                    uint32_t *__restrict__ miss_list, uint32_t *__restrict__ miss_count) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  uint32_t k[8];
  load32(k, L.pk + i * L.pk_stride);
  uint32_t pos;
  const uint32_t found = key_probe<false>(T, k, pos);
  out_vidx[i] = found;
  if (found == HS_NO_KEY) miss_list[atomicAdd(miss_count, 1u)] = (uint32_t)i;  // compacted list for the generic pass
}

// ------------------------------------------------------------------------------------------------ key cache: collect unknown keys
// Copies the key bytes of (up to `max_keys`) records that missed the lookup — or, when nothing is cached yet, of the first
// records of the call — into a compact buffer that is read back asynchronously; the host dedupes them before the NEXT call
// and builds their tables (hs_engine.cu: learn_process).  miss_count == nullptr: take records 0 .. n-1 directly.
__global__ void __launch_bounds__(256) k_gather_keys(in_layout L, size_t n, const uint32_t *__restrict__ miss_list,
                                                     const uint32_t *__restrict__ miss_count, uint32_t max_keys, uint8_t *__restrict__ out_keys,
                                                     uint32_t *__restrict__ out_n) {
  const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
  const size_t avail = miss_count ? (size_t)*miss_count : n;
  const size_t take = avail < max_keys ? avail : max_keys;
  if (t == 0) *out_n = (uint32_t)take;
  if (t >= take) return;
  const size_t i = miss_count ? miss_list[t] : t;
  uint32_t k[8];
  load32(k, L.pk + i * L.pk_stride);
  uint32_t *dst = reinterpret_cast<uint32_t *>(out_keys + t * 32);
#pragma unroll
  for (int j = 0; j < 8; j++) dst[j] = k[j];
}

// ------------------------------------------------------------------------------------------------ phase 1: main
struct main_out {
  fe *xyz;         // 3 field elements per record: X, Y, Z of R' = [S]B + [k](-A)
  uint8_t *meta;   // HS_META_* per record
  int side_pass;   // 1: records without a registered key are handled by the concurrent generic pass
};
struct committee_tables {
  const uint8_t *pks;
  const uint8_t *key_flags;
  uint32_t n_keys;
  const ge_niels *atables;
  size_t table_entries;  // ge_niels per key
};

// Grid-stride over records so the same kernel serves a full launch (one pass) and the compacted miss list, whose length
// only the device knows (n_ptr): no host round trip between the committee pass and the generic pass.
template <bool COMMITTEE>
#ifndef HS_MAIN_MINBLOCKS
#define HS_MAIN_MINBLOCKS 4
#endif
#ifndef HS_GENERIC_MINBLOCKS
#define HS_GENERIC_MINBLOCKS 3
#endif
__global__ void __launch_bounds__(HS_THREADS, COMMITTEE ? HS_MAIN_MINBLOCKS : HS_GENERIC_MINBLOCKS) k_verify_main(in_layout L, size_t n_arg, const uint32_t *__restrict__ n_ptr,
                                                             const uint32_t *__restrict__ index_list, const ge_niels *__restrict__ btable,
                                                             committee_tables C, main_out O, const comb_params cp) {
  // one buffer, two lives: record staging while loading, then the signed digits [digit][thread] (conflict-free columns)
  __shared__ __align__(16) unsigned char smem_raw[HS_MAX_DIGITS * HS_THREADS * 4];
  static_assert(sizeof(smem_raw) >= (HS_THREADS / 32) * 256 * sizeof(uint4), "staging does not fit");
  uint4(*stage)[256] = reinterpret_cast<uint4(*)[256]>(smem_raw);
  int32_t *digits = reinterpret_cast<int32_t *>(smem_raw) + threadIdx.x;
  const size_t n = n_ptr ? (size_t)*n_ptr : n_arg;
  for (size_t base = (size_t)blockIdx.x * blockDim.x; base < n; base += (size_t)gridDim.x * blockDim.x) {  // blockDim <= HS_THREADS
  const size_t t = base + threadIdx.x;
  const size_t warp_first = t & ~(size_t)31;
  // (no early exit for warps past the end: every warp of the block reaches the barriers below; they clamp and do not store)
  const bool active = t < n;
  size_t i = active ? t : n - 1;
  uint32_t R[8], S[8], A[8], h[16];
  uint32_t v = 0;
  bool have_key = true;
  if (L.aos128 && !index_list) {
    uint32_t M[8];
    __syncthreads();  // the previous grid-stride iteration's digits live in the same shared bytes
    warp_load_rec128(R, S, A, M, L.sig, n, warp_first, stage[threadIdx.x >> 5]);
    __syncthreads();
    if (COMMITTEE) {
      v = __ldg(L.vidx + i);
      have_key = v < C.n_keys;
      if (!have_key) v = 0;
      load32(A, C.pks + (size_t)v * 32);  // hash the registered key bytes (identical to the record's on a lookup hit)
    }
    sha512_ram32(h, R, A, M);
  } else {
    if (index_list) i = index_list[i];
    load32(R, L.sig + i * L.sig_stride);
    load32(S, L.sig + i * L.sig_stride + 32);
    if (COMMITTEE) {
      v = __ldg(L.vidx + i);
      have_key = v < C.n_keys;
      if (!have_key) v = 0;
      load32(A, C.pks + (size_t)v * 32);
    } else {
      load32(A, L.pk + i * L.pk_stride);
    }
    const uint8_t *m = L.off ? L.msg + L.off[i] : L.msg + (size_t)(L.midx ? __ldg(L.midx + i) : i) * L.msg_stride;
    const uint64_t len = L.off ? (L.off[i + 1] - L.off[i]) : L.fixed_len;
    if (len == 32 && ((reinterpret_cast<uintptr_t>(m) & 3u) == 0)) {
      uint32_t M[8];
      load32(M, m);
      sha512_ram32(h, R, A, M);
    } else {
      uint64_t pre[8];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        pre[j] = be64_from_le32(R[2 * j], R[2 * j + 1]);
        pre[4 + j] = be64_from_le32(A[2 * j], A[2 * j + 1]);
      }
      sha512_prefix_msg(h, pre, 8, m, len);
    }
  }
  ge_ext acc;
  uint32_t meta;
  if (COMMITTEE) {
    meta = verify_committee_main(acc, R, S, h, btable, C.atables + (size_t)v * C.table_entries, have_key ? C.key_flags[v] : 0u, digits,
                                 HS_THREADS, cp);
    if (!have_key) {
      if (O.side_pass) continue;  // unknown key bytes: the generic pass on the side stream owns this record's outputs
      meta = 0;                   // unknown authority INDEX: reject (messages.rs:57-61 rejects it before any crypto)
    }
  } else {
    ge_cached tab[9];
    meta = verify_generic_main(acc, R, S, A, h, btable, tab, digits, HS_THREADS, cp);
  }
  if (!active) continue;
  if (!(meta & HS_META_PARSE_OK)) {  // keep the batched inversion well-defined for rejected records
    fe_set0(acc.X);
    fe_set1(acc.Y);
    fe_set1(acc.Z);
  }
  uint4 *dst = reinterpret_cast<uint4 *>(O.xyz + i * 3);
  dst[0] = make_uint4(acc.X.v[0], acc.X.v[1], acc.X.v[2], acc.X.v[3]);
  dst[1] = make_uint4(acc.X.v[4], acc.X.v[5], acc.X.v[6], acc.X.v[7]);
  dst[2] = make_uint4(acc.Y.v[0], acc.Y.v[1], acc.Y.v[2], acc.Y.v[3]);
  dst[3] = make_uint4(acc.Y.v[4], acc.Y.v[5], acc.Y.v[6], acc.Y.v[7]);
  dst[4] = make_uint4(acc.Z.v[0], acc.Z.v[1], acc.Z.v[2], acc.Z.v[3]);
  dst[5] = make_uint4(acc.Z.v[4], acc.Z.v[5], acc.Z.v[6], acc.Z.v[7]);
  O.meta[i] = (uint8_t)meta;
  }
}

// ------------------------------------------------------------------------------------------------ latency path (n <= 64)
// One Block::verify / Vote::verify / 3-vote QC of a 4-node deployment is 1 .. 64 signatures (BASELINE config[4]): the
// throughput kernels above would spend 5 launches and ~28 serial mixed additions + an inversion on it (r1: 155 us per
// verify).  Here ONE launch of 64-thread blocks does a signature per block: warp 0 hashes, recodes, lets lane j fetch the table
// entry of digit j and sums the lanes' points with a shuffle tree (5 levels); warp 1 decompresses R meanwhile; thread 0
// compares projectively.  Inputs and verdicts live in mapped pinned host memory (no copy calls).  Registered / cached keys
// only (the host resolves key bytes to indices first).
// One launch serves many REQUESTS (the verify queue coalesces concurrent small verifies): block b takes ring record
// (base + b) & mask, the record names its request slot and the request's record count, and the block that finishes a
// request's last record raises THAT request's completion word — a submitter sees its verdicts when its own records are
// done, not when the launch is.  The synchronous latency path is the one-request case (slot 0, base 0).
struct small_rec {
  uint8_t sig[64];
  uint8_t msg[32];
  uint32_t vidx;
  uint32_t req;    // request slot: index of the request's counter and completion word
  uint32_t req_n;  // records of that request
  uint32_t pad[5];
};
static_assert(sizeof(small_rec) == 128, "small_rec is 128 bytes");
#define HS_SMALL_MAX 64
__device__ __forceinline__ void fe_shfl_down(fe &r, const fe &a, int delta) {
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, a.v[i], delta);
}

// ------------------------------------------------------------------------------------------------ signature cache (hs_queue_sig_cache)
// A queue's table in HBM of the records its kernels accepted under batch-eq: (sig[64] | pk[32] | msg[32]) -> the record's flag
// byte.  The key bytes are the registered key's (C.pks), never its index: hs_committee_update reuses indices.  A record's flags
// depend on these 128 bytes alone, so a hit (all 128 bytes equal) answers both verdict modes exactly and committee changes need
// no flush.  Buckets of HS_SIG_WAYS entries; the bucket is a keyed mix of the 32 record words (a random key per queue, so records
// cannot be aimed at one bucket from outside); a full bucket's victim comes from its round-robin counter.  Each entry is a seqlock:
// seq 0 = never written, odd = being written, even = holds a record.  A writer claims with atomicCAS(seq, even, even + 1), writes,
// fences and stores even + 2; a reader loads seq (acquire), the payload and flags (relaxed, so L1 is bypassed: the other queue
// stream writes too), fences and re-reads seq: a hit needs both reads equal, even, non-zero, and every word equal.
#define HS_SIG_WAYS 4
struct sig_entry {
  uint32_t w[32];  // sig | pk | msg
  uint32_t seq;
  uint32_t flags;
  uint32_t pad[2];
};
static_assert(sizeof(sig_entry) == 144, "sig_entry is 144 bytes");
struct sig_bucket {
  sig_entry e[HS_SIG_WAYS];
  uint32_t rr;  // round-robin victim counter
  uint32_t pad[3];
};
// Counters of a request, summed per block into ctr[4 * slot ..] (slot = the request's ring slot) and moved to the mapped host array
// by the block that completes the request, before its completion word: [0] records probed, [1] hits, [2] inserts, [3] inserts
// that evicted a live entry.
#define HS_SIG_CTRS 4
struct sig_cache_dev {
  sig_bucket *b;        // the table (nullptr when the launch runs without it)
  const uint64_t *key;  // 32 words: the bucket mix's key
  uint32_t bmask;       // buckets - 1
  uint32_t *ctr;        // device: HS_SIG_CTRS per ring slot
  uint32_t *hctr;       // mapped host: the same layout
};
#define HS_SIG_HIT 0x100u  // a probe's result: stored flags | HS_SIG_HIT (0 = miss)

__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu(uint32_t *p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t sig_mix(uint32_t w, uint64_t k) {  // splitmix64's finalizer of (word << 32) ^ key
  uint64_t z = ((uint64_t)w << 32) ^ k;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t sig_bucket_of(const sig_cache_dev &sc, uint64_t h) { return (uint32_t)(h >> 32) & sc.bmask; }
__device__ __forceinline__ uint32_t pick8(const uint32_t (&a)[8], int i) {  // a[i] without local memory
  uint32_t r = a[0];
#pragma unroll
  for (int j = 1; j < 8; j++)
    if (i == j) r = a[j];
  return r;
}
// Warp-wide probe: lane l holds word l of the record.  Every lane must call it; the result is the same on every lane.
__device__ __forceinline__ uint32_t sig_probe_warp(const sig_cache_dev &sc, uint32_t w, int lane, uint32_t &bucket) {
  uint64_t h = sig_mix(w, __ldg(sc.key + lane));
#pragma unroll
  for (int d = 16; d; d >>= 1) h += __shfl_xor_sync(0xffffffffu, h, d);
  bucket = sig_bucket_of(sc, h);
  const sig_entry *x = sc.b[bucket].e;
  uint32_t s0[HS_SIG_WAYS], m[HS_SIG_WAYS], f[HS_SIG_WAYS];
#pragma unroll
  for (int e = 0; e < HS_SIG_WAYS; e++) s0[e] = ld_acquire_gpu(&x[e].seq);
#pragma unroll
  for (int e = 0; e < HS_SIG_WAYS; e++) {
    m[e] = ld_relaxed_gpu(x[e].w + lane);
    f[e] = ld_relaxed_gpu(&x[e].flags);
  }
  __threadfence();
#pragma unroll
  for (int e = 0; e < HS_SIG_WAYS; e++) {
    // each lane read its word between two equal reads of seq; the same even value on every lane makes them one version.  The
    // shuffles stay outside any condition: every lane must reach them.
    const uint32_t s1 = ld_relaxed_gpu(&x[e].seq), s_lane0 = __shfl_sync(0xffffffffu, s0[e], 0), fl = __shfl_sync(0xffffffffu, f[e], 0);
    const bool ok = s0[e] != 0 && !(s0[e] & 1u) && s1 == s0[e] && s0[e] == s_lane0 && m[e] == w;
    if (__all_sync(0xffffffffu, ok)) return fl | HS_SIG_HIT;
  }
  return 0;
}
// One thread's probe of its own record (k_verify_bulk): word(j) = word j of the record.
template <class W>
__device__ __forceinline__ uint32_t sig_probe_thread(const sig_cache_dev &sc, W word, uint32_t &bucket) {
  uint64_t h = 0;
#pragma unroll
  for (int j = 0; j < 32; j++) h += sig_mix(word(j), __ldg(sc.key + j));
  bucket = sig_bucket_of(sc, h);
  const sig_entry *x = sc.b[bucket].e;
#pragma unroll 1
  for (int e = 0; e < HS_SIG_WAYS; e++) {
    const uint32_t s0 = ld_acquire_gpu(&x[e].seq);
    if (!s0 || (s0 & 1u) || ld_relaxed_gpu(x[e].w) != word(0)) continue;
    bool eq = true;
#pragma unroll
    for (int j = 1; j < 32; j++) eq &= ld_relaxed_gpu(x[e].w + j) == word(j);
    const uint32_t fl = ld_relaxed_gpu(&x[e].flags);
    __threadfence();
    if (eq && ld_relaxed_gpu(&x[e].seq) == s0) return fl | HS_SIG_HIT;
  }
  return 0;
}
// One thread inserts an accepted record into its bucket: a never-written entry if there is one, else the round-robin victim.  A
// claim another writer won is retried, at most HS_SIG_WAYS times; then the record is simply not cached.  Returns 0: not inserted,
// 1: inserted into a free entry, 2: inserted over a live entry.
template <class W>
__device__ __forceinline__ uint32_t sig_insert(const sig_cache_dev &sc, uint32_t bucket, W word, uint32_t flags) {
  sig_bucket *b = sc.b + bucket;
#pragma unroll 1
  for (int attempt = 0; attempt < HS_SIG_WAYS; attempt++) {
    int e = -1;
    uint32_t old = 0;
#pragma unroll 1
    for (int i = 0; i < HS_SIG_WAYS && e < 0; i++)
      if (ld_relaxed_gpu(&b->e[i].seq) == 0) e = i;
    if (e < 0) {
      e = (int)(atomicAdd(&b->rr, 1u) % HS_SIG_WAYS);
      old = ld_relaxed_gpu(&b->e[e].seq);
      if (old & 1u) continue;
    }
    sig_entry *x = b->e + e;
    if (atomicCAS(&x->seq, old, old + 1) != old) continue;
    __threadfence();
#pragma unroll
    for (int j = 0; j < 32; j++) st_relaxed_gpu(x->w + j, word(j));
    st_relaxed_gpu(&x->flags, flags);
    __threadfence();
    st_relaxed_gpu(&x->seq, old + 2);
    return old ? 2u : 1u;
  }
  return 0;
}
// A block's counts for request slot `req`, ordered before the block's completion add.
__device__ __forceinline__ void sig_count(const sig_cache_dev &sc, uint32_t req, uint32_t probed, uint32_t hits, uint32_t ins, uint32_t ev) {
  uint32_t *c = sc.ctr + HS_SIG_CTRS * (size_t)req;
  if (probed) atomicAdd(c, probed);
  if (hits) atomicAdd(c + 1, hits);
  if (ins) atomicAdd(c + 2, ins);
  if (ev) atomicAdd(c + 3, ev);
  __threadfence();
}
// The block completing request slot `req` moves its counts to the host and clears them for the slot's next request.
__device__ __forceinline__ void sig_publish(const sig_cache_dev &sc, uint32_t req) {
#pragma unroll
  for (int k = 0; k < HS_SIG_CTRS; k++) sc.hctr[HS_SIG_CTRS * (size_t)req + k] = atomicExch(sc.ctr + HS_SIG_CTRS * (size_t)req + k, 0u);
}
// Per-kernel shared scratch of the cache-on instantiations only (the cache-off kernels keep their shared-memory size).
template <int N>
__device__ __forceinline__ uint32_t *sig_smem() {
  __shared__ __align__(16) uint32_t s[N];
  return s;
}

// Completion step of the queue kernels: k of request slot `req`'s req_n records are done.  Before this add the caller has stored
// those records' flags and fenced them to system scope, and (cache on) added its counts with sig_count, so the add that completes
// the request comes after every record's flags and counts.  That add publishes the cache counts (SIGC), resets the slot's counter
// for its next request, fences to system scope and only then sets the request's completion word to seq.  The queue's watcher
// thread takes that word as its only signal: on seeing it, it reads the request's flags and counts from mapped memory and may hand
// the slot to a new request at once.  req_n is a reference so that a field of the mapped ring is read after the add.
template <bool SIGC>
__device__ __forceinline__ void queue_complete(uint32_t *counters, volatile uint32_t *done, uint32_t seq, uint32_t req, const uint32_t &req_n,
                                               uint32_t k, const sig_cache_dev &sc) {
  if (atomicAdd(counters + req, k) == req_n - k) {
    if constexpr (SIGC) sig_publish(sc, req);
    counters[req] = 0;
    __threadfence_system();
    done[req] = seq;
  }
}

// SIGC: probe and fill the signature cache.  The cache-off instantiation is the kernel without it, instruction for instruction.
template <bool SIGC>
__global__ void __launch_bounds__(64) k_verify_small(const small_rec *__restrict__ ring, uint32_t base, uint32_t mask, const ge_niels *__restrict__ btable,
                                                      committee_tables C, const comb_params cp, uint8_t *out_flags, uint32_t *counters,
                                                      volatile uint32_t *done, uint32_t seq, sig_cache_dev sc) {
  __shared__ int32_t dig[HS_MAX_DIGITS];
  __shared__ fe sh_acc[3], sh_r[2];
  __shared__ uint32_t sh_meta[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t slot = (base + blockIdx.x) & mask;
  const small_rec *rec = ring + slot;
  uint32_t R[8], S[8];
  load32(R, rec->sig);
  load32(S, rec->sig + 32);
  uint32_t v = rec->vidx;
  const bool have_key = v < C.n_keys;
  if (!have_key) v = 0;
  const uint32_t a_flags = have_key ? C.key_flags[v] : 0u;
  uint32_t *sk = nullptr;  // cache on: [0, 32) the record's words, [32] the probe's result, [33] its bucket
  if constexpr (SIGC) {
    sk = sig_smem<34>();
    if (warp == 0) {
      uint32_t hit = 0, bucket = 0;
      if (have_key) {  // slow-path riders (HS_NO_KEY) neither probe nor insert
        uint32_t A[8], M[8];
        load32(A, C.pks + (size_t)v * 32);
        load32(M, rec->msg);
        const int j = lane & 7;
        const uint32_t w = lane < 8 ? pick8(R, j) : lane < 16 ? pick8(S, j) : lane < 24 ? pick8(A, j) : pick8(M, j);
        sk[lane] = w;
        hit = sig_probe_warp(sc, w, lane, bucket);
      }
      if (lane == 0) {
        sk[32] = hit;
        sk[33] = bucket;
      }
    }
    __syncthreads();
    const uint32_t hit = sk[32];
    if (hit) {  // the stored flags, then the counter and completion step; no hashing, no decompression
      if (threadIdx.x == 0) {
        out_flags[slot] = (uint8_t)hit;
        const uint32_t req = rec->req;
        sig_count(sc, req, 1, 1, 0, 0);
        __threadfence_system();
        queue_complete<SIGC>(counters, done, seq, req, rec->req_n, 1u, sc);
      }
      return;
    }
  }
  if (warp == 0) {
    uint32_t A[8], M[8], h[16], k[8];
    load32(A, C.pks + (size_t)v * 32);
    load32(M, rec->msg);
    sha512_ram32(h, R, A, M);
    sc_reduce512(k, h);
    if (lane == 0) {  // one writer for the shared digit array
      sc_digits_rt(dig, 1, k, cp.bias_a, cp.wa, cp.na);
      sc_digits_rt(dig + cp.na, 1, S, cp.bias_b, cp.wb, cp.nb);
    }
    __syncwarp();
    const int NT = cp.na + cp.nb;
    ge_ext acc;
    ge_identity(acc);
#pragma unroll 1
    for (int j = lane; j < NT; j += 32) {  // NT <= 32 for every production geometry: one entry per lane
      uint32_t neg;
      bool is_a;
      const ge_niels *e = comb_entry(C.atables + (size_t)v * C.table_entries, btable, dig, 1, j, cp, neg, is_a);
      niels_signed q;
      niels_load_signed(q, e, neg, false);
      ge_ext p;
      ge_from_signed_niels(p, q.m0, q.m1);
      if (j == lane) acc = p;
      else ge_add_ext(acc, acc, p);
    }
#pragma unroll 1
    for (int step = 1; step < 32; step <<= 1) {
      ge_ext o;
      fe_shfl_down(o.X, acc.X, step);
      fe_shfl_down(o.Y, acc.Y, step);
      fe_shfl_down(o.Z, acc.Z, step);
      fe_shfl_down(o.T, acc.T, step);
      ge_add_ext(acc, acc, o);
    }
    if (lane == 0) {
      sh_acc[0] = acc.X;
      sh_acc[1] = acc.Y;
      sh_acc[2] = acc.Z;
    }
  } else {
    ge_ext Rpt;
    const uint32_t r_ok = ge_decompress(Rpt, R);
    const uint32_t parse_ok = sc_is_canonical(S) & a_flags & 1u & (have_key ? 1u : 0u);
    const uint32_t small = ge_enc_is_small_order(R) | ((a_flags >> 1) & 1u);
    if (lane == 0) {
      sh_r[0] = Rpt.X;
      sh_r[1] = Rpt.Y;
      sh_meta[0] = parse_ok & r_ok;
      sh_meta[1] = (parse_ok ? HS_F_PARSE_OK : 0u) | (small ? HS_F_SMALL : 0u);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t fl = sh_meta[1];
    const uint32_t eq = sh_meta[0] & ge_proj_equals_affine(sh_acc[0], sh_acc[1], sh_acc[2], sh_r[0], sh_r[1]);
    if (eq) fl |= HS_F_EQ;
    if (eq && !(fl & HS_F_SMALL)) fl |= HS_F_STRICT;
    out_flags[slot] = (uint8_t)fl;
    if constexpr (SIGC) {
      const uint32_t ins = (have_key && (fl & HS_F_EQ)) ? sig_insert(sc, sk[33], [&](int j) { return sk[j]; }, fl) : 0u;
      sig_count(sc, rec->req, have_key ? 1u : 0u, 0, ins != 0, ins == 2);
    }
    __threadfence_system();
    queue_complete<SIGC>(counters, done, seq, rec->req, rec->req_n, 1u, sc);
  }
}

// ------------------------------------------------------------------------------------------------ block-wide inversion
// Montgomery's trick over a block of 128 threads: tot[t] becomes 1 / tot[t].  Lane l of warp 0 multiplies tot[4l .. 4l+3], inverts
// that product once and back-substitutes.  Every tot[t] must be nonzero.  The caller takes a barrier before (tot stored) and after
// (tot read back).
__device__ __forceinline__ void block_invert4(fe (&tot)[128]) {
  if (threadIdx.x < 32) {
    const int b = threadIdx.x * 4;
    fe q0 = tot[b], q1, q2, q3, inv, u;
    fe_mul(q1, q0, tot[b + 1]);
    fe_mul(q2, q1, tot[b + 2]);
    fe_mul(q3, q2, tot[b + 3]);
    fe_invert(inv, q3);
    fe_mul(u, inv, q2);        // 1 / tot[b+3]
    fe_mul(inv, inv, tot[b + 3]);
    tot[b + 3] = u;
    fe_mul(u, inv, q1);        // 1 / tot[b+2]
    fe_mul(inv, inv, tot[b + 2]);
    tot[b + 2] = u;
    fe_mul(u, inv, q0);        // 1 / tot[b+1]
    fe_mul(inv, inv, tot[b + 1]);
    tot[b + 1] = u;
    tot[b] = inv;              // 1 / tot[b]
  }
}
// A zero Z cannot come from a curve point.  Setting it to 1 and clearing the record's parse bit keeps one bad record from poisoning
// the block's shared inversion.
__device__ __forceinline__ void guard_zero_z(fe &Z, uint32_t &meta) {
  if (fe_is_zero(Z)) {
    fe_set1(Z);
    meta &= ~HS_META_PARSE_OK;
  }
}

// ------------------------------------------------------------------------------------------------ bulk queue path (large groups)
// A certificate of a large committee (thousands of votes) as ONE queue request: k_verify_small would spend a 64-thread block and a
// square-root chain on every signature, several waves of them.  Here a THREAD verifies a signature as k_verify_main<true> does,
// straight from the queue's mapped ring (logical record i = ring slot (base + i) & mask, so a group may wrap the ring's end), and
// the block finishes its own records: the block's Z's share one batched inversion (block_invert4), then the affine comparison with
// R's encoding — no decompression of R, no global scratch, no second launch.  Flags and completion as in k_verify_small: both HS_F_EQ and HS_F_STRICT
// per record, one counter add per block, and the block that completes the request raises its completion word.  One launch carries
// exactly one request (n records).
// Sizing: 128 threads, at least 3 blocks per SM.  R and the request fields stay live across the comb, so the 4-block budget of
// k_verify_main (128 registers) spilled; 3 blocks allow 168 (sm_90a: 142 registers, 0 spills, 36,864 bytes smem).  A 6,668-record
// certificate is 53 blocks, one per SM, so occupancy does not bound this launch at committee sizes.
// SIGC (signature cache on): each thread probes its own record first; a hit skips the hash and the comb but still takes part in
// every barrier (Z = 1 in the block's inversion) and writes the stored flags; a miss that verifies under batch-eq is inserted.  S, A
// and M wait for the insert in shared memory (12 KB more: 48 KB, the static limit), so they need not stay live across the comb.
#define HS_BULK_THREADS 128
#define HS_BULK_MINBLOCKS 3
template <bool SIGC>
__global__ void __launch_bounds__(HS_BULK_THREADS, HS_BULK_MINBLOCKS) k_verify_bulk(const small_rec *__restrict__ ring, uint32_t base, uint32_t mask,
                                                                                  uint32_t n, const ge_niels *__restrict__ btable, committee_tables C,
                                                                                  const comb_params cp, uint8_t *out_flags, uint32_t *counters,
                                                                                  volatile uint32_t *done, uint32_t seq, sig_cache_dev sc) {
  // one buffer, two lives: record staging while loading, then the signed digits [digit][thread] (conflict-free columns)
  __shared__ __align__(16) unsigned char smem_raw[HS_MAX_DIGITS * HS_BULK_THREADS * 4];
  static_assert(sizeof(smem_raw) >= (HS_BULK_THREADS / 32) * 256 * sizeof(uint4), "staging does not fit");
  __shared__ fe tot[HS_BULK_THREADS];
  const int lane = threadIdx.x & 31;
  const uint32_t first = blockIdx.x * HS_BULK_THREADS, t = first + threadIdx.x;
  const uint32_t cnt = (n - first < HS_BULK_THREADS) ? n - first : HS_BULK_THREADS;  // records of this block (the last one is partial)
  // (threads past n compute on a zero record and store nothing: every thread reaches the barriers below)
  uint4 q[8];
  uint4 *sw = reinterpret_cast<uint4 *>(smem_raw) + (threadIdx.x >> 5) * 256;
  const uint32_t warp_first = first + (threadIdx.x & ~31u);
  warp_stage_rows128(q, n, warp_first, [&](int r) { return reinterpret_cast<const uint4 *>(ring + ((base + warp_first + r) & mask)); }, sw, lane);
  __syncthreads();  // the staging bytes become the digit slots
  uint32_t R[8], S[8], A[8], h[16];
  unpack8(R, q[0], q[1]);
  unpack8(S, q[2], q[3]);
  uint32_t v = q[6].x;  // small_rec: sig | msg | vidx | req | req_n
  const uint32_t req = q[6].y, req_n = q[6].z;
  const bool have_key = v < C.n_keys;  // HS_NO_KEY (cannot reach this path: kept as in k_verify_small) rejects the record
  if (!have_key) v = 0;
  // cache on: record word j >= 8 of thread t (S, A, M) at keep[((j - 8) / 4 * HS_BULK_THREADS + t) * 4 + j % 4]; R stays in
  // registers across the comb anyway (verify_flags_from reads it)
  uint32_t *keep = nullptr;
  uint32_t hit = 0, bucket = 0;
  const bool probed = SIGC && have_key && threadIdx.x < cnt;
  {
    uint32_t M[8];
    unpack8(M, q[4], q[5]);
    load32(A, C.pks + (size_t)v * 32);  // hash the registered key bytes, as k_verify_main<true>
    if constexpr (SIGC) {
      keep = sig_smem<24 * HS_BULK_THREADS>();
      uint4 *k4 = reinterpret_cast<uint4 *>(keep) + threadIdx.x;
      k4[0] = q[2];
      k4[HS_BULK_THREADS] = q[3];
      k4[2 * HS_BULK_THREADS] = make_uint4(A[0], A[1], A[2], A[3]);
      k4[3 * HS_BULK_THREADS] = make_uint4(A[4], A[5], A[6], A[7]);
      k4[4 * HS_BULK_THREADS] = q[4];
      k4[5 * HS_BULK_THREADS] = q[5];
      if (probed)
        hit = sig_probe_thread(
            sc, [&](int j) { return j < 8 ? R[j] : j < 16 ? S[j - 8] : j < 24 ? A[j - 16] : M[j - 24]; }, bucket);
    }
    if (!hit) sha512_ram32(h, R, A, M);
  }
  ge_ext acc;
  uint32_t meta = 0;
  if (!hit) {
    meta = verify_committee_main(acc, R, S, h, btable, C.atables + (size_t)v * C.table_entries, have_key ? C.key_flags[v] : 0u,
                                 reinterpret_cast<int32_t *>(smem_raw) + threadIdx.x, HS_BULK_THREADS, cp);
  } else {
    fe_set0(acc.X);
    fe_set0(acc.Y);
    fe_set1(acc.Z);
  }
  if (!have_key) meta = 0;
  guard_zero_z(acc.Z, meta);
  tot[threadIdx.x] = acc.Z;
  __syncthreads();
  block_invert4(tot);
  if constexpr (SIGC) {  // the digit slots are free now (every thread is past the comb): word 0 gathers the block's counts
    if (threadIdx.x == 0) *reinterpret_cast<uint32_t *>(smem_raw) = 0;
  }
  __syncthreads();
  uint32_t ins = 0;
  if (threadIdx.x < cnt) {
    const uint32_t fl = hit ? (hit & 0xffu) : verify_flags_from(acc.X, acc.Y, tot[threadIdx.x], R, meta);
    out_flags[(base + t) & mask] = (uint8_t)fl;
    if constexpr (SIGC) {
      if (probed && !hit && (fl & HS_F_EQ))
        ins = sig_insert(
            sc, bucket, [&](int j) { return j < 8 ? R[j] : keep[(((j - 8) >> 2) * HS_BULK_THREADS + threadIdx.x) * 4 + (j & 3)]; }, fl);
    }
    __threadfence_system();
  }
  if constexpr (SIGC) {  // the block's counts, a byte each (at most 128), summed per warp and then in shared memory: one barrier
    uint32_t *sum = reinterpret_cast<uint32_t *>(smem_raw);
    const uint32_t w = __reduce_add_sync(0xffffffffu, (probed ? 1u : 0u) | (hit ? 1u << 8 : 0u) | (ins ? 1u << 16 : 0u) | (ins == 2 ? 1u << 24 : 0u));
    if (lane == 0) atomicAdd(sum, w);
    __syncthreads();
    if (threadIdx.x == 0) sig_count(sc, req, *sum & 0xffu, (*sum >> 8) & 0xffu, (*sum >> 16) & 0xffu, *sum >> 24);
  } else {
    __syncthreads();
  }
  if (threadIdx.x == 0) queue_complete<SIGC>(counters, done, seq, req, req_n, cnt, sc);  // thread 0 holds a record of the request
}

// ------------------------------------------------------------------------------------------------ generic queue path (hs_queue_generic)
// Queue requests the committee path cannot serve (no committee registered, or a key outside it), verified on the GPU instead of on
// the dispatcher thread.  One launch carries every such request of one or more dispatches: record j is ring slot slots[(first + j)
// & mask] (a mapped list the dispatcher writes), its key the 32 bytes at pks + 32 * slot (the queue's mapped key array).  A thread
// verifies a record as k_verify_main<false> does: SHA-512(R || A || M), decompress A, a radix-16 window for [k](-A) from a per-thread
// table of 8 multiples, the base comb for [S]B; then, as k_verify_bulk, the block's Z's share one inversion and verify_flags_from
// writes both HS_F_EQ and HS_F_STRICT.  A block may hold records of several requests (and a request may span blocks), so completion
// counts records: the add that completes a request fences the system and raises its completion word.  Rows are staged as in
// k_verify_bulk, a warp's 32 records with 16-byte loads: each record's 128 bytes are one coalesced row wherever its slot is.
// Sizing: 128 threads, 3 blocks per SM as k_verify_main<false> (the window table is per-thread local memory, not a spill).
#define HS_GEN_THREADS 128
__global__ void __launch_bounds__(HS_GEN_THREADS, HS_GENERIC_MINBLOCKS) k_queue_generic(const small_rec *__restrict__ ring, const uint8_t *__restrict__ pks,
                                                                                      const uint32_t *__restrict__ slots, uint32_t first, uint32_t mask,
                                                                                      uint32_t n, const ge_niels *__restrict__ btable, const comb_params cp,
                                                                                      uint8_t *out_flags, uint32_t *counters, volatile uint32_t *done,
                                                                                      uint32_t seq) {
  // one buffer, two lives: record staging while loading, then the base comb's signed digits [digit][thread]
  __shared__ __align__(16) unsigned char smem_raw[HS_MAX_DIGITS * HS_GEN_THREADS * 4];
  static_assert(sizeof(smem_raw) >= (HS_GEN_THREADS / 32) * 256 * sizeof(uint4), "staging does not fit");
  __shared__ fe tot[HS_GEN_THREADS];
  const int lane = threadIdx.x & 31;
  const uint32_t j = blockIdx.x * HS_GEN_THREADS + threadIdx.x;
  const bool active = j < n;  // threads past n take every barrier with Z = 1 and store nothing
  const uint32_t slot = active ? __ldg(slots + ((first + j) & mask)) : 0u;
  uint4 q[8];
  uint4 *sw = reinterpret_cast<uint4 *>(smem_raw) + (threadIdx.x >> 5) * 256;
  warp_stage_rows128(q, n, j & ~31u, [&](int r) { return reinterpret_cast<const uint4 *>(ring + __shfl_sync(0xffffffffu, slot, r)); }, sw, lane);
  __syncthreads();  // the staging bytes become the digit slots
  uint32_t R[8];
  unpack8(R, q[0], q[1]);
  const uint32_t req = q[6].y, req_n = q[6].z;  // small_rec: sig | msg | vidx | req | req_n
  ge_ext acc;
  uint32_t meta = 0;
  if (active) {
    uint32_t S[8], A[8], M[8], h[16];
    unpack8(S, q[2], q[3]);
    unpack8(M, q[4], q[5]);
    const uint4 *a4 = reinterpret_cast<const uint4 *>(pks + 32 * (size_t)slot);
    unpack8(A, __ldg(a4), __ldg(a4 + 1));
    sha512_ram32(h, R, A, M);
    ge_cached tab[9];
    meta = verify_generic_main(acc, R, S, A, h, btable, tab, reinterpret_cast<int32_t *>(smem_raw) + threadIdx.x, HS_GEN_THREADS, cp);
  }
  if (!(meta & HS_META_PARSE_OK)) {  // rejected records (and idle threads) keep the block's inversion well-defined
    fe_set0(acc.X);
    fe_set1(acc.Y);
    fe_set1(acc.Z);
  }
  guard_zero_z(acc.Z, meta);
  tot[threadIdx.x] = acc.Z;
  __syncthreads();
  block_invert4(tot);
  __syncthreads();
  if (!active) return;
  out_flags[slot] = (uint8_t)verify_flags_from(acc.X, acc.Y, tot[threadIdx.x], R, meta);
  __threadfence_system();
  queue_complete<false>(counters, done, seq, req, req_n, 1u, {});
}

// A few LONG messages (one mempool batch is ~15 kB = 120 blocks, mempool/src/processor.rs:30): SHA-512 is sequential in its
// 80 x nblk rounds, but the message schedule (45 % of the work) of different blocks is independent — lane l of the warp
// expands block g + l into a shared K+W table, then the rounds run back to back from that table.  One warp per message.
__global__ void __launch_bounds__(32) k_digest32_long(const uint8_t *__restrict__ data, const uint64_t *__restrict__ off, size_t n,
                                                       uint32_t *__restrict__ out) {
  __shared__ uint64_t kw[80 * 32];
  const size_t i = blockIdx.x;
  if (i >= n) return;
  const int lane = threadIdx.x;
  const uint8_t *m = data + off[i];
  const uint64_t len = off[i + 1] - off[i];
  const uint64_t nblk = sha512_nblocks(len);
  sha512_state s;
  sha512_init(s);
#pragma unroll 1
  for (uint64_t g0 = 0; g0 < nblk; g0 += 32) {
    if (g0 + lane < nblk) {
      uint64_t w[16];
      sha512_block_words(w, m, len, g0 + lane);
      sha512_expand_kw(kw + lane, 32, w);
    }
    __syncwarp();
    const int cnt = (int)((nblk - g0 < 32) ? (nblk - g0) : 32);
#pragma unroll 1
    for (int j = 0; j < cnt; j++) sha512_compress_kw_strided(s, kw + j, 32);  // every lane runs the same rounds (broadcast reads)
    __syncwarp();
  }
  if (lane == 0) {
    uint32_t h[16];
    sha512_output_words(s, h);
    store_digest32(out + i * 8, h);
  }
}

// ------------------------------------------------------------------------------------------------ multi-GPU epilogue
// The accept bitmap of a sharded verify has to reach every rank (each validator process needs every verdict).  Instead of a
// separate all-gather collective after the kernel, the finish kernel stores each bitmap word it produces straight into EVERY
// peer's result buffer over NVLink (P2P stores through CUDA-IPC mapped pointers), then a release flag per (writer, reader)
// pair tells the reader the shard has landed.  Payload is n/8 bytes per rank: latency, not bandwidth.
#define HS_MAX_PEERS 16
// Result buffer of one rank (cudaMalloc'd, exported over CUDA IPC):
//   [2][total_words]  the global bitmap, double-buffered by epoch parity: a fast rank's epoch e+1 words land in the OTHER
//                     half, so a slower rank that is still reading epoch e never sees them (r1's single buffer had a
//                     write-after-read hazard); a rank can run at most one epoch ahead, because finishing epoch e+1
//                     needs every peer's epoch e+1 flag, which a peer publishes only after its own epoch-e readers ran
//                     (stream order: consume epoch e's bitmap before enqueueing the verify of epoch e+1)
//   [HS_MAX_PEERS]    flags[w] = last epoch whose words from writer w have landed here (release/acquire, system scope)
//   [0] timeout flag, [1] finish-kernel block counter
struct peer_route {
  uint32_t *buf[HS_MAX_PEERS];  // buf[p] = base of rank p's result buffer as mapped in THIS process
  int n;                        // world size (0 = route disabled: plain local bitmap)
  int my_rank;
  uint32_t epoch;
  size_t total_words;           // words of the global bitmap; rank p owns [p * total_words / n, (p + 1) * total_words / n)
  size_t word_offset;           // this rank's first word in the global bitmap
};
#define HS_PEER_FLAGS(P) ((P).total_words * 2)
#define HS_PEER_CTRL(P) ((P).total_words * 2 + HS_MAX_PEERS)
// Executed by ONE block after all of this rank's words of the epoch are stored (and fenced): thread p publishes this rank's
// flag in rank p's buffer, then waits for rank p's flag here.  A peer that never shows up is an error, not a hang: the spin
// is bounded, the sticky timeout flag is raised and that peer's shard is cleared (every verdict reads "reject").
__device__ __forceinline__ void peer_signal_and_wait(const peer_route &P) {
  const int p = threadIdx.x;
  if (p >= P.n) return;
  uint32_t *own = P.buf[P.my_rank];
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(P.buf[p] + HS_PEER_FLAGS(P) + P.my_rank), "r"(P.epoch) : "memory");
  uint32_t v = 0;
  bool ok = false;
  for (long long spin = 0; spin < (1ll << 24); spin++) {  // bounded (~5 s)
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(own + HS_PEER_FLAGS(P) + p) : "memory");
    if ((int32_t)(v - P.epoch) >= 0) {
      ok = true;
      break;
    }
    __nanosleep(200);
  }
  if (!ok) {
    own[HS_PEER_CTRL(P)] = 1;
    const size_t per = P.total_words / P.n;
    uint32_t *w = own + (P.epoch & 1u) * P.total_words + (size_t)p * per;
    for (size_t k = 0; k < per; k++) w[k] = 0;
  }
}
// shard without records: nothing to verify, but the peers still wait for this rank's flag
__global__ void k_peer_sync_only(const peer_route P) { peer_signal_and_wait(P); }

// ------------------------------------------------------------------------------------------------ phase 2: finish
__device__ __forceinline__ void fe_load_global(fe &r, const fe *p) {
  const uint4 *s = reinterpret_cast<const uint4 *>(p);
  unpack8(r.v, s[0], s[1]);
}
// One thread owns `group` (16, 8 or 4: fewer for small batches, so that enough blocks exist to hide the one serial field inversion
// each block waits for — at 126 k records the 16-record form ran 62 blocks for 110 us) consecutive records.  Montgomery's trick at two levels so that ONE
// field inversion per 64 records is executed (by warp 0, lane l inverting the product of threads 4l..4l+3) instead of one
// per thread: phase A prefix products of the thread's 16 Z's; phase B the block-level inversion through shared memory;
// phase C back-substitution + affine comparison with R's encoding.  Two neighbouring lanes combine their 16 verdicts into
// one bitmap word, which goes to the local bitmap or — armed by hs_peer_next — straight into every peer's buffer, after
// which the last block of the grid exchanges the epoch flags with the peers (no separate signal / wait launches).
// The verify flag that decides a record's verdict in `mode`: HS_MODE_BATCH_EQ selects HS_F_EQ, any other value HS_F_STRICT (the
// host entry points reject values above 1; device mode bytes are not checked).
__host__ __device__ inline uint32_t mode_flag(uint32_t mode) { return mode == HS_MODE_BATCH_EQ ? HS_F_EQ : HS_F_STRICT; }
// verdict(i, fl) turns record i's flags into its bit: one mode for the pass (k_verify_finish) or record i's own mode byte
// (k_verify_finish_modes).
// CACHED (a pass that shares a queue's signature cache, hs_queue_sig_share): a record k_sig_probe decided carries HS_META_CACHED and
// its stored flags in meta and Z = 1 in xyz, so it takes its flags from meta; every record's flag byte goes to fl_out for k_sig_fill.
// The CACHED = false instantiations are the kernels without it, instruction for instruction.
#define HS_META_CACHED 0x40u  // meta: decided from the signature cache; the low bits are the stored flags
template <bool CACHED, class Verdict>
__device__ __forceinline__ void verify_finish_body(const in_layout &L, size_t n, const fe *__restrict__ xyz, const uint8_t *__restrict__ meta,
                                                   Verdict verdict, uint32_t *__restrict__ bitmap, const peer_route &P, const int group,
                                                   uint8_t *__restrict__ fl_out = nullptr) {
  __shared__ fe tot[HS_THREADS];
  const size_t t = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  const size_t first = t * (size_t)group;
  const int cnt = (first < n) ? (int)((n - first < (size_t)group) ? (n - first) : group) : 0;
  fe prod[HS_FINISH_GROUP];
  fe run;
  fe_set1(run);
#pragma unroll 1
  for (int c = 0; c < cnt; c++) {
    fe Z;
    fe_load_global(Z, xyz + (first + c) * 3 + 2);
    if (fe_is_zero(Z)) fe_set1(Z);  // cannot happen for curve points; keeps one bad record from poisoning the group
    fe_mul(run, run, Z);
    prod[c] = run;
  }
  tot[threadIdx.x] = run;
  __syncthreads();
  block_invert4(tot);
  __syncthreads();
  uint32_t bits = 0;
  if (cnt) {
    fe u = tot[threadIdx.x];
#pragma unroll 1
    for (int c = cnt - 1; c >= 0; c--) {
      const size_t i = first + c;
      fe X, Y, Z, zinv;
      fe_load_global(X, xyz + i * 3 + 0);
      fe_load_global(Y, xyz + i * 3 + 1);
      fe_load_global(Z, xyz + i * 3 + 2);
      const uint32_t zero_z = fe_is_zero(Z);
      if (zero_z) fe_set1(Z);
      if (c > 0) fe_mul(zinv, u, prod[c - 1]);
      else zinv = u;
      fe_mul(u, u, Z);
      uint32_t R[8];
      load32(R, L.sig + i * L.sig_stride);
      uint32_t m = meta[i];
      if (zero_z) m &= ~HS_META_PARSE_OK;
      uint32_t fl;
      if constexpr (CACHED) {
        fl = (m & HS_META_CACHED) ? (m & 0x1fu) : verify_flags_from(X, Y, zinv, R, m);
        fl_out[i] = (uint8_t)fl;
      } else {
        fl = verify_flags_from(X, Y, zinv, R, m);
      }
      const uint32_t ok = verdict(i, fl);
      if (ok) bits |= 1u << c;
    }
  }
  // 32 / group neighbouring lanes hold the verdicts of one bitmap word: butterfly-OR them together
  const int lanes_per_word = 32 / group;
  uint32_t word = bits << (group * (threadIdx.x & (lanes_per_word - 1)));
  for (int m = 1; m < lanes_per_word; m <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, m);
  if ((threadIdx.x & (lanes_per_word - 1)) == 0 && first < n) {
    const size_t widx = t / lanes_per_word;
    if (P.n == 0) {
      bitmap[widx] = word;
    } else {
      const size_t at = (P.epoch & 1u) * P.total_words + P.word_offset + widx;
#pragma unroll 1
      for (int p = 0; p < P.n; p++) P.buf[p][at] = word;  // fused all-gather: one NVLink store per peer
    }
  }
  if (P.n) {
    // the last block to get here publishes the epoch flag to every peer and waits for theirs: the exchange costs no launch
    __shared__ int is_last;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(P.buf[P.my_rank] + HS_PEER_CTRL(P) + 1, 1u) == gridDim.x - 1;
    __syncthreads();
    if (is_last) {
      peer_signal_and_wait(P);
      __syncthreads();
      if (threadIdx.x == 0) P.buf[P.my_rank][HS_PEER_CTRL(P) + 1] = 0;
    }
  }
}
__global__ void __launch_bounds__(HS_THREADS) k_verify_finish(in_layout L, size_t n, const fe *__restrict__ xyz, const uint8_t *__restrict__ meta,
                                                               uint32_t mode, uint32_t *__restrict__ bitmap, const peer_route P, const int group) {
  verify_finish_body<false>(L, n, xyz, meta, [&](size_t, uint32_t fl) { return fl & mode_flag(mode); }, bitmap, P, group);
}
// Per-record verdict modes (hs_verify_groups_dev, hs_verify_groups, the queue's batch lane): every word written locally or stored into
// the peers' buffers is a final item verdict.
__global__ void __launch_bounds__(HS_THREADS) k_verify_finish_modes(in_layout L, size_t n, const fe *__restrict__ xyz, const uint8_t *__restrict__ meta,
                                                                     const uint8_t *__restrict__ item_mode, uint32_t *__restrict__ bitmap, const peer_route P,
                                                                     const int group) {
  verify_finish_body<false>(L, n, xyz, meta, [&](size_t i, uint32_t fl) { return fl & mode_flag(item_mode[i]); }, bitmap, P, group);
}
// The same two kernels for a pass that shares a signature cache (CACHED above).
__global__ void __launch_bounds__(HS_THREADS) k_verify_finish_cached(in_layout L, size_t n, const fe *__restrict__ xyz, const uint8_t *__restrict__ meta,
                                                                      uint32_t mode, uint32_t *__restrict__ bitmap, const peer_route P, const int group,
                                                                      uint8_t *__restrict__ fl_out) {
  verify_finish_body<true>(L, n, xyz, meta, [&](size_t, uint32_t fl) { return fl & mode_flag(mode); }, bitmap, P, group, fl_out);
}
__global__ void __launch_bounds__(HS_THREADS) k_verify_finish_modes_cached(in_layout L, size_t n, const fe *__restrict__ xyz,
                                                                            const uint8_t *__restrict__ meta, const uint8_t *__restrict__ item_mode,
                                                                            uint32_t *__restrict__ bitmap, const peer_route P, const int group,
                                                                            uint8_t *__restrict__ fl_out) {
  verify_finish_body<true>(L, n, xyz, meta, [&](size_t i, uint32_t fl) { return fl & mode_flag(item_mode[i]); }, bitmap, P, group, fl_out);
}

// ------------------------------------------------------------------------------------------------ shared signature cache (hs_queue_sig_share)
// A synchronous verify pass or a batch-lane pass that shares a queue's signature cache runs k_sig_probe after the key lookup,
// k_verify_main<committee> over the records it left, the cached finish kernel, then k_sig_fill.  Counts go to sc.ctr: [0] records
// probed, [1] hits (k_sig_probe), [2] inserts, [3] inserts that evicted a live entry (k_sig_fill).  Only records with a registered key
// and a 32-byte message (every pass that shares has one) take part; the words of record i are sig | registered key bytes | Digest.
struct sig_rec_words {
  uint32_t R[8], S[8], A[8], M[8];
  __device__ __forceinline__ uint32_t operator()(int j) const { return j < 8 ? R[j] : j < 16 ? S[j - 8] : j < 24 ? A[j - 16] : M[j - 24]; }
};
__device__ __forceinline__ void sig_load_words(sig_rec_words &w, const in_layout &L, const committee_tables &C, size_t i, uint32_t v) {
  load32(w.R, L.sig + i * L.sig_stride);
  load32(w.S, L.sig + i * L.sig_stride + 32);
  load32(w.A, C.pks + (size_t)v * 32);
  load32(w.M, L.msg + (size_t)(L.midx ? __ldg(L.midx + i) : i) * L.msg_stride);
}
// The block's counts into two of sc.ctr's words: per warp with one reduction each, then one atomic per warp.
__device__ __forceinline__ void sig_count_pair(const sig_cache_dev &sc, int k, uint32_t a, uint32_t b) {
  const uint32_t sa = __reduce_add_sync(0xffffffffu, a), sb = __reduce_add_sync(0xffffffffu, b);
  if ((threadIdx.x & 31) == 0) {
    if (sa) atomicAdd(sc.ctr + k, sa);
    if (sb) atomicAdd(sc.ctr + k + 1, sb);
  }
}
// One thread per record.  A hit writes the stored flags | HS_META_CACHED to meta and (0 : 1 : 1) to xyz, so the finish kernel's inversion
// stays well-defined; every other record the committee pass owns is appended to list (count in *list_n), warp by warp in record order.
// With side_pass, records whose key missed the lookup belong to the generic pass and are left alone.  Only a slot in service (flag bit 0,
// which k_verify_main<true> requires for acceptance) is probed: hs_committee_update's removal and hs_table_repair's rebuild clear only a
// slot's flags, so its old key bytes stay in C.pks and would still match a record cached before; such a record goes to the list instead
// and is rejected there, as without the cache.
__global__ void __launch_bounds__(256) k_sig_probe(in_layout L, size_t n, committee_tables C, sig_cache_dev sc, int side_pass, fe *__restrict__ xyz,
                                                   uint8_t *__restrict__ meta, uint32_t *__restrict__ list, uint32_t *__restrict__ list_n) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  const bool active = i < n;
  const uint32_t v = active ? __ldg(L.vidx + i) : HS_NO_KEY;
  const bool have_key = v < C.n_keys;
  const bool in_service = have_key && (__ldg(C.key_flags + v) & 1u);
  uint32_t hit = 0;
  if (in_service) {
    sig_rec_words w;
    sig_load_words(w, L, C, i, v);
    uint32_t bucket;
    hit = sig_probe_thread(sc, w, bucket);
  }
  if (hit) {
    meta[i] = (uint8_t)((hit & 0x1fu) | HS_META_CACHED);
    uint4 *dst = reinterpret_cast<uint4 *>(xyz + i * 3);
    dst[0] = dst[1] = dst[3] = dst[5] = make_uint4(0, 0, 0, 0);
    dst[2] = dst[4] = make_uint4(1, 0, 0, 0);
  }
  const bool append = active && !hit && (have_key || !side_pass);
  const uint32_t mask = __ballot_sync(0xffffffffu, append);
  const int lane = threadIdx.x & 31;
  uint32_t base = 0;
  if (mask && lane == 0) base = atomicAdd(list_n, (uint32_t)__popc(mask));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (append) list[base + __popc(mask & ((1u << lane) - 1u))] = (uint32_t)i;
  sig_count_pair(sc, 0, in_service ? 1u : 0u, hit ? 1u : 0u);
}
// One thread per record: a record the pass verified (not decided from the cache) with a registered key, judged strict (by its mode
// byte, else the pass's mode) and with HS_F_EQ in its flags fl[i] is inserted with its whole flag byte.
__global__ void __launch_bounds__(256) k_sig_fill(in_layout L, size_t n, committee_tables C, sig_cache_dev sc, const uint8_t *__restrict__ meta,
                                                  const uint8_t *__restrict__ fl, uint32_t mode, const uint8_t *__restrict__ item_mode) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  uint32_t ins = 0;
  if (i < n) {
    const uint32_t v = __ldg(L.vidx + i), f = fl[i];
    const bool strict = mode_flag(item_mode ? item_mode[i] : mode) == HS_F_STRICT;
    if (v < C.n_keys && !(meta[i] & HS_META_CACHED) && strict && (f & HS_F_EQ)) {
      sig_rec_words w;
      sig_load_words(w, L, C, i, v);
      uint64_t h = 0;
#pragma unroll
      for (int j = 0; j < 32; j++) h += sig_mix(w(j), __ldg(sc.key + j));
      ins = sig_insert(sc, sig_bucket_of(sc, h), w, f);
    }
  }
  sig_count_pair(sc, 2, ins != 0, ins == 2);
}
// The audit of a signature-cache table (hs_queue_sig_audit): a thread per entry of buckets [first, first + count), grid-stride.  An entry
// read as one version by the probes' rule (seq acquired, the words and flags relaxed, a fence, seq again) is re-checked from its 128 bytes
// alone with explain_record, which reads no table; flags_from_why of the result is the byte any verify path writes for that record.  An
// entry whose byte differs gets that byte through sig_insert's writer protocol (claim seq, store, fence, release s0 + 2), so a hit
// answers exactly what a verify would, reject included.  seq never goes back to 0 and the words are never cleared: 128 zero bytes are
// a record too.  An entry being written, torn between the reads, or claimed by a writer before the correction is skipped.
// out: [0] held, [1] corrected, [2] skipped, [3] the first correction as position (bucket * HS_SIG_WAYS + way) << 24 | stored byte << 16 |
// derived byte << 8 | why, kept by atomicMin (position < 2^26).
__global__ void __launch_bounds__(HS_THREADS) k_sig_audit(sig_bucket *b, uint32_t first, uint32_t count, unsigned long long *out) {
  uint32_t held = 0, corrected = 0, skipped = 0;
  for (uint32_t j = blockIdx.x * HS_THREADS + threadIdx.x; j < count * HS_SIG_WAYS; j += gridDim.x * HS_THREADS) {
    const uint32_t bucket = first + j / HS_SIG_WAYS, way = j % HS_SIG_WAYS;
    sig_entry *x = b[bucket].e + way;
    const uint32_t s0 = ld_acquire_gpu(&x->seq);
    if (!s0) continue;
    uint32_t R[8], S[8], A[8], M[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      R[k] = ld_relaxed_gpu(x->w + k);
      S[k] = ld_relaxed_gpu(x->w + 8 + k);
      A[k] = ld_relaxed_gpu(x->w + 16 + k);
      M[k] = ld_relaxed_gpu(x->w + 24 + k);
    }
    const uint32_t fl = ld_relaxed_gpu(&x->flags);
    __threadfence();
    if ((s0 & 1u) || ld_relaxed_gpu(&x->seq) != s0) {
      skipped++;
      continue;
    }
    uint32_t h[16];
    sha512_ram32(h, R, A, M);
    ge_cached tab[9];
    const uint32_t why = explain_record(R, S, A, h, tab), want = flags_from_why(why);
    if ((fl & 0x1fu) == want) {
      held++;
      continue;
    }
    if (atomicCAS(&x->seq, s0, s0 + 1) != s0) {  // a writer put a newer record here
      skipped++;
      continue;
    }
    __threadfence();
    st_relaxed_gpu(&x->flags, want);
    __threadfence();
    st_relaxed_gpu(&x->seq, s0 + 2);
    held++;
    corrected++;
    atomicMin(out + 3, ((unsigned long long)(bucket * HS_SIG_WAYS + way) << 24) | ((fl & 0xffu) << 16) | (want << 8) | why);
  }
  held = __reduce_add_sync(0xffffffffu, held);
  corrected = __reduce_add_sync(0xffffffffu, corrected);
  skipped = __reduce_add_sync(0xffffffffu, skipped);
  if ((threadIdx.x & 31) == 0) {
    if (held) atomicAdd(out, (unsigned long long)held);
    if (corrected) atomicAdd(out + 1, (unsigned long long)corrected);
    if (skipped) atomicAdd(out + 2, (unsigned long long)skipped);
  }
}

// ------------------------------------------------------------------------------------------------ table construction
// thread = (point p, window w, block b of HS_BUILD_BLOCK entries).  slots (nullable): point p is slot slots[p], its key at encs + 32
// slots[p] and its table at slot slots[p] of `tables`; its flag byte still goes to key_flags[p].  Without a list, slot p.
#define HS_BUILD_BLOCK 64
__global__ void __launch_bounds__(HS_THREADS) k_build_comb(const uint8_t *__restrict__ encs, const uint32_t *__restrict__ slots, size_t n_points,
                                                            int negate, int W, int n_windows, ge_niels *tables, uint8_t *key_flags) {
  const int entries = 1 << (W - 1);
  const int blocks_per_window = entries / HS_BUILD_BLOCK;
  const size_t t = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  const size_t per_point = (size_t)n_windows * blocks_per_window;
  const size_t p = t / per_point;
  if (p >= n_points) return;
  const size_t s = slots ? slots[p] : p;
  const int w = (int)((t % per_point) / blocks_per_window);
  const int b = (int)(t % blocks_per_window);
  ge_ext P;
  if (encs) {
    uint32_t e[8];
    load32(e, encs + s * 32);
    uint32_t ok = ge_decompress(P, e);
    uint32_t small = ge_enc_is_small_order(e);
    if (w == 0 && b == 0 && key_flags) key_flags[p] = (uint8_t)((ok & 1u) | (small << 1));
    if (!ok) ge_identity(P);  // the table of a rejected key is never used for an accept (flag bit0 = 0)
  } else {
    ge_basepoint(P);
  }
  if (negate) {
    ge_ext Q;
    ge_neg(Q, P);
    P = Q;
  }
  fe prod[HS_BUILD_BLOCK];
  comb_build_block(tables + s * ((size_t)n_windows * comb_window_stride(W)), P, W, w, b * HS_BUILD_BLOCK, HS_BUILD_BLOCK, prod);
}

// ------------------------------------------------------------------------------------------------ table audit (hs_table_audit)
// Findings: HS_AUDIT_* bits OR-ed into bits[0] (the base table), bits[1] (hash entries naming no slot in use) and bits[2 + s] (slot s),
// and the first finding's audit_key() kept by an atomic minimum, so the message does not depend on scheduling.
struct audit_out {
  unsigned long long *first;
  uint32_t *bits;
};
__device__ __forceinline__ void audit_report(const audit_out &O, size_t bits_idx, uint32_t cls, uint64_t key) {
  atomicOr(O.bits + bits_idx, cls);
  atomicMin(O.first, (unsigned long long)key);
}
// KEY / FLAG / LOOKUP: thread i < n_slots checks slot i, thread n_slots + j checks hash entry j.  live: the engine's liveness mirror
// (1 byte per slot); expect_pks / expect_live: the caller's map (nullable).  Writes auditable[s] = live and the key decompresses: the
// slots whose comb table k_table_audit then checks.
__global__ void __launch_bounds__(256) k_slot_audit(key_table T, const uint8_t *__restrict__ key_flags, const uint8_t *__restrict__ live,
                                                    const uint8_t *__restrict__ expect_pks, const uint32_t *__restrict__ expect_live, int expect,
                                                    uint8_t *__restrict__ auditable, audit_out O) {
  const size_t n_slots = T.n_keys;
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i < n_slots) {
    const uint32_t is_live = live[i] ? 1u : 0u;
    uint32_t k[8];
    load32(k, T.pks + i * 32);
    uint32_t cls = 0;
    if (expect) {
      const uint32_t want_live = expect_live ? (expect_live[i >> 5] >> (i & 31)) & 1u : 1u;
      if (want_live != is_live) cls |= HS_AUDIT_KEY;
      if (expect_pks && is_live && want_live) {
        uint32_t e[8], d = 0;
        load32(e, expect_pks + i * 32);
#pragma unroll
        for (int j = 0; j < 8; j++) d |= e[j] ^ k[j];
        if (d) cls |= HS_AUDIT_KEY;
      }
    }
    ge_ext P;
    const uint32_t ok = ge_decompress(P, k);
    const uint32_t want_flag = is_live ? (ok | (ge_enc_is_small_order(k) << 1)) : 0u;
    if (key_flags[i] != want_flag) cls |= HS_AUDIT_FLAG;
    if (is_live) {
      uint32_t pos;
      const uint32_t idx = key_probe<true>(T, k, pos);
      if (idx == HS_NO_KEY || !live[idx]) cls |= HS_AUDIT_LOOKUP;
    }
    auditable[i] = (uint8_t)(is_live & ok);
    if (cls) audit_report(O, 2 + i, cls, audit_key(i + 1, 0, 0));
  } else if (i - n_slots <= T.mask) {
    const uint32_t j = (uint32_t)(i - n_slots), idx = T.slots[j];
    if (idx == HS_NO_KEY) return;
    if (idx >= n_slots) {
      audit_report(O, 1, HS_AUDIT_LOOKUP, audit_key(n_slots + 1, 0, 0));
      return;
    }
    uint32_t k[8], pos = HS_NO_KEY;
    load32(k, T.pks + (size_t)idx * 32);
    if (!live[idx] || key_probe<true>(T, k, pos) != idx || pos != j) audit_report(O, 2 + idx, HS_AUDIT_LOOKUP, audit_key(idx + 1, 0, 0));
  }
}
// TABLE / BASE: a warp per run of 32 consecutive entries of one window of one table, lane l entry first + l (coalesced 96-byte loads);
// entry m - 1 comes from lane l - 1 by shuffles, and entry 1 of the window is one broadcast load.  The lane of entry 1 also checks the
// window link, or for window 0 the anchor.  pks == nullptr: one table, the base-point table (anchor B); otherwise table s is slot s's,
// anchored on -A of its stored bytes, and only the slots k_slot_audit marked auditable are read.  LISTED: table t is slot slots[t]'s
// (key bytes and table), with auditable[t] and the findings at list position t; otherwise slot t's, and `slots` is not read (the full
// audit keeps the code it had before the list).  Short blocks: the lowest-priority stream's blocks give way to verify launches at every
// block boundary.
#define HS_AUDIT_WARPS 4
// The window findings of the mend's audits (hs_table_mend), by audit_mend_flags: bit base + t (n_windows + 1) + i for window i of table
// t (its list position, slot or 0 for the base-point table), and bit base + t (n_windows + 1) + n_windows when its anchor failed.
struct audit_wins {
  uint32_t *bits;
  uint64_t base;
};
__device__ __forceinline__ void audit_report_windows(const audit_wins &Wo, uint64_t t, uint32_t win, int n_windows, uint32_t f) {
  const uint64_t row = Wo.base + t * (uint64_t)(n_windows + 1);
  const auto set = [&](uint64_t b) { atomicOr(Wo.bits + (b >> 5), 1u << (b & 31)); };
  if (f & 1u) set(row + win);
  if (f & 2u) set(row + win - 1);
  if (f & 4u) set(row + n_windows);
}
// The body of both table forms; WINDOWS also reports the windows to mend (the kernels without it keep the code they had before).
template <bool LISTED, bool WINDOWS>
__device__ __forceinline__ void table_audit_run(const ge_niels *__restrict__ tables, const uint32_t *__restrict__ slots, size_t n_tables,
                                                size_t table_entries, int W, int n_windows, const uint8_t *__restrict__ pks,
                                                const uint8_t *__restrict__ auditable, const audit_out &O, const audit_wins &Wo) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t H = (uint64_t)1 << (W - 1), runs = (H + 1 + 31) / 32;
  const uint64_t g = (uint64_t)blockIdx.x * HS_AUDIT_WARPS + (threadIdx.x >> 5);
  const uint64_t t = g / (runs * n_windows);
  if (t >= n_tables || (pks && !auditable[t])) return;  // whole warps leave together
  const uint64_t s = LISTED ? slots[t] : t;
  const uint32_t win = (uint32_t)((g / runs) % n_windows);
  const uint32_t m = (uint32_t)((g % runs) * 32 + lane);
  const ge_niels *wt = tables + s * table_entries + (size_t)win * comb_window_stride(W);
  const bool in = m <= H;
  ge_niels e, prev, one;
  niels_load_stream(e, wt + (in ? m : H));
  niels_load(one, wt + 1);
  {
    uint32_t *pe = reinterpret_cast<uint32_t *>(&e), *pp = reinterpret_cast<uint32_t *>(&prev);
#pragma unroll
    for (int j = 0; j < 24; j++) pp[j] = __shfl_up_sync(0xffffffffu, pe[j], 1);
  }
  if (lane == 0 && m > 0) niels_load(prev, wt + m - 1);
  uint32_t ok = in ? audit_entry_local(e, prev, one, m) : 1u;
  uint32_t edge = 1u;  // the anchor or link check, apart from ok in the WINDOWS form
  if (m == 1) {
    if (win == 0) {
      ge_ext P;
      audit_anchor_point(P, pks ? reinterpret_cast<const uint32_t *>(pks + s * 32) : nullptr);
      if constexpr (WINDOWS) edge = audit_anchor(e, P);
      else ok &= audit_anchor(e, P);
    } else {
      ge_niels last;
      niels_load(last, wt - comb_window_stride(W) + H);
      if constexpr (WINDOWS) edge = audit_link(e, last);
      else ok &= audit_link(e, last);
    }
  }
  if constexpr (WINDOWS) {
    if (!(ok & edge)) audit_report(O, pks ? 2 + t : 0, pks ? HS_AUDIT_TABLE : HS_AUDIT_BASE, audit_key(pks ? t + 1 : 0, win + 1, m));
    audit_report_windows(Wo, t, win, n_windows, audit_mend_flags(win, m, ok, edge));
  } else if (!ok) {
    audit_report(O, pks ? 2 + t : 0, pks ? HS_AUDIT_TABLE : HS_AUDIT_BASE, audit_key(pks ? t + 1 : 0, win + 1, m));
  }
}
template <bool LISTED>
__global__ void __launch_bounds__(32 * HS_AUDIT_WARPS) k_table_audit(const ge_niels *__restrict__ tables, const uint32_t *__restrict__ slots,
                                                                       size_t n_tables, size_t table_entries, int W, int n_windows,
                                                                       const uint8_t *__restrict__ pks, const uint8_t *__restrict__ auditable,
                                                                       audit_out O) {
  table_audit_run<LISTED, false>(tables, slots, n_tables, table_entries, W, n_windows, pks, auditable, O, audit_wins{});
}
// The same with the window findings (hs_table_mend's audits).
template <bool LISTED>
__global__ void __launch_bounds__(32 * HS_AUDIT_WARPS) k_table_audit(const ge_niels *__restrict__ tables, const uint32_t *__restrict__ slots,
                                                                       size_t n_tables, size_t table_entries, int W, int n_windows,
                                                                       const uint8_t *__restrict__ pks, const uint8_t *__restrict__ auditable,
                                                                       audit_out O, audit_wins Wo) {
  table_audit_run<LISTED, true>(tables, slots, n_tables, table_entries, W, n_windows, pks, auditable, O, Wo);
}
// The range form (hs_scrub_start): entries [first, first + count) of the base-point table, entry e being entry e % (2^(W-1) + 1) of
// window e / (2^(W-1) + 1), the table's storage order.  Warp g takes the g-th run of 32 entries of one window from the run holding
// `first`, with the checks above; a lane outside the range only feeds the shuffles.  An entry's checks read its own window and, for
// entry 1, entry 2^(W-1) of the window before, so slices that together cover the table find exactly what the full audit finds, and
// report it with the same key.  An overload of the unlisted form, so the two forms above keep their code.
template <bool WINDOWS>
__device__ __forceinline__ void table_audit_range_run(const ge_niels *__restrict__ tables, uint64_t first, uint64_t count, int W, int n_windows,
                                                      const audit_out &O, const audit_wins &Wo) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t H = (uint64_t)1 << (W - 1), stride = H + 1, runs = (H + 1 + 31) / 32;
  const uint64_t r = (first / stride) * runs + (first % stride) / 32 + (uint64_t)blockIdx.x * HS_AUDIT_WARPS + (threadIdx.x >> 5);
  const uint64_t win = r / runs;
  if (win >= (uint64_t)n_windows) return;  // whole warps leave together
  const uint32_t m = (uint32_t)((r % runs) * 32 + lane);
  const uint64_t idx = win * stride + m;
  const bool in_window = m <= H, in = in_window && idx >= first && idx - first < count;
  if (!__any_sync(0xffffffffu, in)) return;
  const ge_niels *wt = tables + win * stride;
  ge_niels e, prev, one;
  niels_load_stream(e, wt + (in_window ? m : H));
  niels_load(one, wt + 1);
  {
    uint32_t *pe = reinterpret_cast<uint32_t *>(&e), *pp = reinterpret_cast<uint32_t *>(&prev);
#pragma unroll
    for (int j = 0; j < 24; j++) pp[j] = __shfl_up_sync(0xffffffffu, pe[j], 1);
  }
  if (lane == 0 && m > 0) niels_load(prev, wt + m - 1);
  uint32_t ok = in ? audit_entry_local(e, prev, one, m) : 1u;
  uint32_t edge = 1u;  // the anchor or link check, apart from ok in the WINDOWS form
  if (in && m == 1) {
    if (win == 0) {
      ge_ext P;
      audit_anchor_point(P, nullptr);
      if constexpr (WINDOWS) edge = audit_anchor(e, P);
      else ok &= audit_anchor(e, P);
    } else {
      ge_niels last;
      niels_load(last, wt - stride + H);
      if constexpr (WINDOWS) edge = audit_link(e, last);
      else ok &= audit_link(e, last);
    }
  }
  if constexpr (WINDOWS) {
    if (!(ok & edge)) audit_report(O, 0, HS_AUDIT_BASE, audit_key(0, (uint32_t)win + 1, m));
    audit_report_windows(Wo, 0, (uint32_t)win, n_windows, audit_mend_flags((uint32_t)win, m, ok, edge));
  } else if (!ok) {
    audit_report(O, 0, HS_AUDIT_BASE, audit_key(0, (uint32_t)win + 1, m));
  }
}
template <bool LISTED>
__global__ void __launch_bounds__(32 * HS_AUDIT_WARPS) k_table_audit(const ge_niels *__restrict__ tables, uint64_t first, uint64_t count,
                                                                       int W, int n_windows, audit_out O) {
  static_assert(!LISTED, "the range form covers the base-point table");
  table_audit_range_run<false>(tables, first, count, W, n_windows, O, audit_wins{});
}
template <bool LISTED>
__global__ void __launch_bounds__(32 * HS_AUDIT_WARPS) k_table_audit(const ge_niels *__restrict__ tables, uint64_t first, uint64_t count,
                                                                       int W, int n_windows, audit_out O, audit_wins Wo) {
  static_assert(!LISTED, "the range form covers the base-point table");
  table_audit_range_run<true>(tables, first, count, W, n_windows, O, Wo);
}

// ------------------------------------------------------------------------------------------------ mend (hs_table_mend)
// A work item: window `win` of the base-point table (slot == HS_MEND_BASE) or of slot `slot`'s comb table.
#define HS_MEND_BASE 0xffffffffu
struct mend_item {
  uint32_t slot, win;
};
// thread = (item, block b of HS_BUILD_BLOCK entries of its window), blocks [first_block, first_block + n_blocks) of the launch's items
// in (item, b) order.  Each thread builds its block into its own HS_BUILD_BLOCK + 1 entries of `stage` (comb_mend_block: the arithmetic
// of k_build_comb, P = -A from the slot's stored key bytes or B) and stores the entries that differ from the live table.  rewritten:
// the entries stored, reduced per warp.  A key that does not decompress has no table to mend (the audit does not check it either).
__global__ void __launch_bounds__(HS_THREADS) k_mend_windows(const mend_item *__restrict__ items, uint64_t first_block, uint64_t n_blocks, int W,
                                                             ge_niels *tables, size_t table_entries, const uint8_t *__restrict__ pks,
                                                             ge_niels *stage, unsigned long long *rewritten) {
  const uint64_t t = (uint64_t)blockIdx.x * HS_THREADS + threadIdx.x;
  const uint64_t blocks_per_window = ((uint64_t)1 << (W - 1)) / HS_BUILD_BLOCK;
  uint32_t stored = 0;
  if (t < n_blocks) {
    const uint64_t g = first_block + t;
    const mend_item it = items[g / blocks_per_window];
    const int b = (int)(g % blocks_per_window);
    const bool base = it.slot == HS_MEND_BASE;
    ge_ext P;
    if (audit_anchor_point(P, base ? nullptr : reinterpret_cast<const uint32_t *>(pks + 32 * (size_t)it.slot))) {
      ge_niels *window = tables + (base ? 0 : it.slot * table_entries) + (size_t)it.win * comb_window_stride(W);
      fe prod[HS_BUILD_BLOCK];
      stored = comb_mend_block(window, stage + t * (HS_BUILD_BLOCK + 1), P, W, (int)it.win, b * HS_BUILD_BLOCK, HS_BUILD_BLOCK, prod);
    }
  }
  stored = __reduce_add_sync(0xffffffffu, stored);
  if ((threadIdx.x & 31) == 0 && stored) atomicAdd(rewritten, (unsigned long long)stored);
}

// ------------------------------------------------------------------------------------------------ explanation of a verdict
// hs_explain_rec128: a thread per packed hs_rec128 record, grid-stride, one HS_WHY_* byte out per record.  It reads the records and
// nothing else (explain_record is table-free), and loads them with its own plain per-thread loads: it runs on rejected records only.
__global__ void __launch_bounds__(HS_THREADS) k_explain(const uint8_t *__restrict__ recs, size_t n, uint8_t *__restrict__ out_why) {
  for (size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * HS_THREADS) {
    const uint8_t *r = recs + i * 128;
    uint32_t R[8], S[8], A[8], M[8], h[16];
    load32(R, r);
    load32(S, r + 32);
    load32(A, r + 64);
    load32(M, r + 96);
    sha512_ram32(h, R, A, M);
    ge_cached tab[9];
    out_why[i] = (uint8_t)explain_record(R, S, A, h, tab);
  }
}

// The verify queue's explain lane (hs_queue_submit_explain, hs_queue_submit_explain_msgs).  A request's region of the lane's mapped
// arena is recs (n x 128 B: sig | pk | Digest, the Digest field unused for a preimage request) | pre_off (u64, m + 1) | msg_idx (u32, n)
// | the m preimages | why bytes (n) | tail: [0] records done (in the device mirror), [1] completion word.  A Digest request (m = 0) has
// no preimage sections.  Every section starts 16-byte aligned.
struct xq_layout {
  uint64_t o_off, o_mi, o_pre, o_why, o_tail, size;
};
__host__ __device__ inline xq_layout xq_layout_of(uint64_t n, uint64_t m, uint64_t pre_bytes) {
  auto al = [](uint64_t x) { return (x + 15) & ~(uint64_t)15; };
  xq_layout L;
  L.o_off = 128 * n;
  L.o_mi = L.o_off + (m ? al(8 * (m + 1)) : 0);
  L.o_pre = L.o_mi + (m ? al(4 * n) : 0);
  L.o_why = L.o_pre + al(pre_bytes);
  L.o_tail = L.o_why + al(n);
  L.size = L.o_tail + 16;
  return L;
}
// One explain launch's requests, in submit order: request k's records are the launch's records [first, first + n).
struct xq_desc {
  uint64_t off;        // region offset in the arena (and in its device mirror)
  uint32_t n, first;   // records; index of its record 0 in the launch
  uint32_t m;          // preimages (0: a Digest request)
  uint32_t pre_bytes;  // preimage bytes
  uint32_t seq;        // the completion word's value
  uint32_t pad;
};
static_assert(sizeof(xq_desc) == 32, "xq_desc is 32 bytes");
// A thread per record, grid-stride over the launch's n records (the grid is a fixed share of the SMs: see launch_queue_explain).  The
// thread finds its request in the descriptor list, reads its record from the region's device mirror, hashes its preimage with
// sha512_prefix_msg when it has one (Digest = SHA-512(preimage)[..32]) and runs explain_record exactly as k_explain does.  Its why byte
// goes to the mapped arena; the add that completes a request fences to system scope and raises the request's completion word.  It reads
// the regions and nothing else: no context table, key slot, flag or hash table, and no base-point table.
__global__ void __launch_bounds__(HS_THREADS) k_queue_explain(const xq_desc *__restrict__ list, uint32_t n_desc, uint32_t n,
                                                              uint8_t *mirror, uint8_t *arena) {
  for (uint32_t j = blockIdx.x * HS_THREADS + threadIdx.x; j < n; j += gridDim.x * HS_THREADS) {
    uint32_t lo = 0, hi = n_desc;  // the last request whose first record is <= j
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (list[mid].first <= j) lo = mid;
      else hi = mid;
    }
    const xq_desc d = list[lo];
    const xq_layout L = xq_layout_of(d.n, d.m, d.pre_bytes);
    const uint32_t i = j - d.first;
    uint8_t *reg = mirror + d.off;
    const uint8_t *r = reg + 128 * (size_t)i;
    uint32_t R[8], S[8], A[8], M[8], h[16];
    load32(R, r);
    load32(S, r + 32);
    load32(A, r + 64);
    if (d.m) {
      const uint64_t *pre_off = reinterpret_cast<const uint64_t *>(reg + L.o_off);
      const uint32_t k = reinterpret_cast<const uint32_t *>(reg + L.o_mi)[i];
      const uint64_t none[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      sha512_prefix_msg(h, none, 0, reg + L.o_pre + pre_off[k], pre_off[k + 1] - pre_off[k]);
#pragma unroll
      for (int w = 0; w < 8; w++) M[w] = h[w];
    } else {
      load32(M, r + 96);
    }
    sha512_ram32(h, R, A, M);
    ge_cached tab[9];
    arena[d.off + L.o_why + i] = (uint8_t)explain_record(R, S, A, h, tab);
    __threadfence_system();
    if (atomicAdd(reinterpret_cast<uint32_t *>(reg + L.o_tail), 1u) == d.n - 1) {
      __threadfence_system();
      reinterpret_cast<volatile uint32_t *>(arena + d.off + L.o_tail)[1] = d.seq;
    }
  }
}

// hs_explain_groups_dev: the ordered selection of the items whose bit is 0, then a re-check per selected item.  The selection keeps its
// count on the device: k_sel_count sums the zero bits of each block of HS_SEL_WORDS bitmap words, k_sel_top turns the block sums into
// exclusive offsets (one block, carry across chunks) and writes the counts to out, and k_sel_scatter ranks each word within its block
// again and writes the lowest `cap` indices (explain_select.cuh).  k_explain_items reads its count from out[1].
#define HS_SEL_TOP 1024
// Exclusive prefix sum of v over the block, and the block's total in *total (blockDim.x = HS_SEL_WORDS or HS_SEL_TOP).
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *warp_sums, uint32_t *total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= (uint32_t)d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t s = lane < n_warps ? warp_sums[lane] : 0, t = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, t, d);
      if (lane >= (uint32_t)d) t += y;
    }
    if (lane < n_warps) warp_sums[lane] = t - s;  // exclusive offset of each warp
    if (lane == 31) *total = t;
  }
  __syncthreads();
  const uint32_t r = warp_sums[warp] + x - v;
  __syncthreads();  // warp_sums and *total may be reused by the caller's next scan
  return r;
}
__global__ void __launch_bounds__(HS_SEL_WORDS) k_sel_count(const uint32_t *__restrict__ bm, uint64_t n, uint32_t *__restrict__ bsum) {
  __shared__ uint32_t ws[HS_SEL_WORDS / 32], total;
  const uint64_t w = (uint64_t)blockIdx.x * HS_SEL_WORDS + threadIdx.x;
  const uint32_t c = w < (n + 31) / 32 ? __popc(bitmap_zero_bits(bm[w], n, w)) : 0;
  block_excl_scan(c, ws, &total);
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}
// bsum[0 .. n_blocks) in place -> exclusive offsets.  out: [0] zero bits, [1] selected = min(zero bits, cap), [2] 0 faults, [3] no fault
// yet.
__global__ void __launch_bounds__(HS_SEL_TOP) k_sel_top(uint32_t *bsum, uint32_t n_blocks, uint64_t cap, uint32_t *out) {
  __shared__ uint32_t ws[HS_SEL_TOP / 32], total;
  uint32_t carry = 0;
  for (uint32_t base = 0; base < n_blocks; base += HS_SEL_TOP) {
    const uint32_t b = base + threadIdx.x, v = b < n_blocks ? bsum[b] : 0;
    const uint32_t r = block_excl_scan(v, ws, &total);
    if (b < n_blocks) bsum[b] = carry + r;
    carry += total;
  }
  if (threadIdx.x == 0) {
    out[0] = carry;
    out[1] = cap < carry ? (uint32_t)cap : carry;
    out[2] = 0;
    out[3] = 0xffffffffu;
  }
}
__global__ void __launch_bounds__(HS_SEL_WORDS) k_sel_scatter(const uint32_t *__restrict__ bm, uint64_t n, const uint32_t *__restrict__ boff,
                                                              const uint32_t *__restrict__ out, uint32_t *__restrict__ list) {
  __shared__ uint32_t ws[HS_SEL_WORDS / 32], total;
  const uint64_t w = (uint64_t)blockIdx.x * HS_SEL_WORDS + threadIdx.x;
  const uint32_t zeros = w < (n + 31) / 32 ? bitmap_zero_bits(bm[w], n, w) : 0;
  const uint32_t r = block_excl_scan(__popc(zeros), ws, &total);
  select_scatter(zeros, (uint64_t)boff[blockIdx.x] + r, w, out[1], list);
}
// A thread per selected item, grid-stride over out[1] of them (the grid is a fixed share of the SMs: see launch_explain_items).  Item i
// = list[j] is re-checked exactly as k_queue_explain re-checks a preimage record: sig[i], pk[i] and Digest = SHA-512(preimage of
// msg_idx[i])[..32], hashed by sha512_prefix_msg; then sha512_ram32 and explain_record.  Its why byte goes to why[i]; an item the mask
// finds valid in its mode (why_valid_in_mode) is an engine fault, counted per warp into out[2] with the lowest index in out[3].  It reads
// the caller's arrays and nothing else: no context table, key slot, flag or hash table, and no base-point table.
__global__ void __launch_bounds__(HS_THREADS) k_explain_items(const uint32_t *__restrict__ list, const uint8_t *__restrict__ pre,
                                                              const uint64_t *__restrict__ pre_off, const uint8_t *__restrict__ sig,
                                                              const uint8_t *__restrict__ pk, const uint32_t *__restrict__ msg_idx,
                                                              const uint8_t *__restrict__ mode, uint8_t *__restrict__ why, uint32_t *out) {
  const uint32_t n = out[1];
  uint32_t faults = 0, first = 0xffffffffu;
  for (uint32_t j = blockIdx.x * HS_THREADS + threadIdx.x; j < n; j += gridDim.x * HS_THREADS) {
    const uint32_t i = list[j];
    uint32_t R[8], S[8], A[8], M[8], h[16];
    load32(R, sig + 64 * (size_t)i);
    load32(S, sig + 64 * (size_t)i + 32);
    load32(A, pk + 32 * (size_t)i);
    const uint32_t k = msg_idx[i];
    const uint64_t none[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    sha512_prefix_msg(h, none, 0, pre + pre_off[k], pre_off[k + 1] - pre_off[k]);
#pragma unroll
    for (int w = 0; w < 8; w++) M[w] = h[w];
    sha512_ram32(h, R, A, M);
    ge_cached tab[9];
    const uint32_t y = explain_record(R, S, A, h, tab);
    why[i] = (uint8_t)y;
    if (why_valid_in_mode(y, mode ? mode[i] : HS_MODE_STRICT)) {
      faults++;
      first = min(first, i);
    }
  }
  faults = __reduce_add_sync(0xffffffffu, faults);
  first = __reduce_min_sync(0xffffffffu, first);
  if ((threadIdx.x & 31) == 0 && faults) {
    atomicAdd(out + 2, faults);
    atomicMin(out + 3, first);
  }
}

// ------------------------------------------------------------------------------------------------ Digest kernels
__global__ void __launch_bounds__(HS_THREADS) k_digest32(const uint8_t *__restrict__ data, const uint64_t *__restrict__ off, uint64_t fixed_len,
                                                          size_t n, uint32_t *__restrict__ out) {
  const size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  if (i >= n) return;
  uint32_t h[16];
  uint64_t pre[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const uint8_t *m = off ? data + off[i] : data + i * fixed_len;
  const uint64_t len = off ? off[i + 1] - off[i] : fixed_len;
  sha512_prefix_msg(h, pre, 0, m, len);
  store_digest32(out + i * 8, h);
}

// Verify queue requests that carry signed preimages instead of Digests (hs_queue_submit_msgs).  A request's region of the queue's
// mapped arena is pre_off[m + 1] (u64, relative to the preimage bytes) | msg_idx[n] (u32) | the m preimages, each section 16-byte
// aligned.  The host keeps only the preimages some record names, so each of the m is hashed once.
struct qmsg_desc {
  uint32_t off;        // arena offset of the request's region (16-byte aligned)
  uint32_t m;          // preimages
  uint32_t n;          // records
  uint32_t base;       // ring slot of record 0: record i is slot (base + i) & mask
  uint32_t pre_bytes;  // preimage bytes
  uint32_t pad[3];
};
static_assert(sizeof(qmsg_desc) == 32, "qmsg_desc is 32 bytes");
__host__ __device__ inline uint64_t qmsg_o_pre(uint64_t m, uint64_t n) { return (8 * (m + 1) + 4 * n + 15) & ~(uint64_t)15; }
__host__ __device__ inline uint64_t qmsg_bytes(uint64_t m, uint64_t n, uint64_t pre_bytes) { return qmsg_o_pre(m, n) + ((pre_bytes + 15) & ~(uint64_t)15); }
// One block per preimage request of the launch that follows on the same stream; its descriptor is list[(first + blockIdx.x) & mask].
// The region crosses the bus once (coalesced 16-byte loads into `stage`, the arena's device mirror), each preimage is hashed once
// into the request's digest slots (digs: 32 bytes per 8 arena bytes, so concurrent requests never share one), and every record's
// 32-byte Digest is stored into the msg field of its ring record, where the verify kernel reads it.
#define HS_QDIG_THREADS 256
__global__ void __launch_bounds__(HS_QDIG_THREADS) k_queue_digests(const qmsg_desc *__restrict__ list, uint32_t first, uint32_t mask,
                                                                    const uint8_t *__restrict__ arena, uint8_t *stage, uint32_t *digs, small_rec *ring) {
  const qmsg_desc d = list[(first + blockIdx.x) & mask];
  const uint32_t words = (uint32_t)(qmsg_bytes(d.m, d.n, d.pre_bytes) / 16);
  const uint4 *src = reinterpret_cast<const uint4 *>(arena + d.off);
  uint4 *dst = reinterpret_cast<uint4 *>(stage + d.off);
  for (uint32_t k = threadIdx.x; k < words; k += HS_QDIG_THREADS) dst[k] = src[k];
  __syncthreads();
  const uint64_t *pre_off = reinterpret_cast<const uint64_t *>(stage + d.off);
  const uint32_t *msg_idx = reinterpret_cast<const uint32_t *>(stage + d.off + 8 * ((size_t)d.m + 1));
  const uint8_t *pre = stage + d.off + qmsg_o_pre(d.m, d.n);
  uint32_t *dig = digs + (size_t)(d.off / 8) * 8;
#pragma unroll 1
  for (uint32_t j = threadIdx.x; j < d.m; j += HS_QDIG_THREADS) {
    uint32_t h[16];
    const uint64_t none[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    sha512_prefix_msg(h, none, 0, pre + pre_off[j], pre_off[j + 1] - pre_off[j]);
    store_digest32(dig + (size_t)j * 8, h);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < d.n; i += HS_QDIG_THREADS) {
    const uint4 *s = reinterpret_cast<const uint4 *>(dig + (size_t)msg_idx[i] * 8);
    uint4 *r = reinterpret_cast<uint4 *>(ring[(d.base + i) & mask].msg);
    r[0] = s[0];
    r[1] = s[1];
  }
}

// Fixed-size, 16-byte aligned messages (the transaction / payload shape of BASELINE config[1]): every full 128-byte block is
// fetched by the warp with coalesced 16-byte loads through shared memory (a per-thread 8-byte walk touches 32 sectors per
// load instruction), and when the length is a multiple of 128 the padding-only last block runs without its message
// schedule (sha512_compress_kw).  Other lengths finish through the generic reader.
__global__ void __launch_bounds__(HS_THREADS) k_digest32_fixed(const uint8_t *__restrict__ data, uint64_t len, size_t n, uint32_t *__restrict__ out,
                                                                const sha512_kw padkw, int pad_is_const) {
  __shared__ __align__(16) uint4 stage[HS_THREADS / 32][256];
  const size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  const size_t warp_first = i & ~(size_t)31;
  if (warp_first >= n) return;  // whole warp past the end
  sha512_state s;
  sha512_init(s);
  const uint64_t nfull = len >> 7;
#pragma unroll 1
  for (uint64_t b = 0; b < nfull; b++) {
    uint4 q[8];
    warp_stage_rows128(q, n, warp_first, [&](int r) { return reinterpret_cast<const uint4 *>(data + b * 128 + (warp_first + r) * len); },
                       stage[threadIdx.x >> 5], threadIdx.x & 31);
    __syncwarp();  // the next block is staged into the same rows
    uint64_t w[16];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      w[2 * k] = be64_from_le32(q[k].x, q[k].y);
      w[2 * k + 1] = be64_from_le32(q[k].z, q[k].w);
    }
    sha512_compress(s, w);
  }
  if (i >= n) return;
  if (pad_is_const) {
    sha512_compress_kw(s, padkw);
  } else {
    const uint64_t pre[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    sha512_absorb_blocks(s, pre, 0, data + i * len, len, nfull, sha512_nblocks(len));
  }
  uint32_t h[16];
  sha512_output_words(s, h);
  store_digest32(out + i * 8, h);
}

// ------------------------------------------------------------------------------------------------ per-QC AND
// word w of an all-ones bitmap over n bits (unused high bits of the last word 0)
template <class T>
__host__ __device__ inline uint32_t bitmap_word_ones(const T &n, const T &w) {
  return ((n & 31) && w == (n + 31) / 32 - 1) ? ((1u << (n & 31)) - 1u) : 0xffffffffu;
}
// vote i belongs to certificate qc_idx[i]; a rejected vote clears its certificate's bit (qc bitmap pre-set to all ones)
__global__ void __launch_bounds__(256) k_qc_and(const uint32_t *__restrict__ vote_bitmap, const uint32_t *__restrict__ qc_idx, size_t n_votes,
                                                size_t n_qc, uint32_t *__restrict__ qc_bitmap) {
  const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n_votes) return;
  if (!((vote_bitmap[i >> 5] >> (i & 31)) & 1u)) {
    const uint32_t j = qc_idx[i];
    if (j < n_qc) atomicAnd(qc_bitmap + (j >> 5), ~(1u << (j & 31)));
  }
}

// Completion of a verify-queue batch pass (hs_queue_submit_batch), in place of k_qc_and + copies + a stream synchronise: item i's
// verdict is bit i of `items` (k_verify_finish_modes); the item bits are balloted straight into the request's mapped result words
// (after the group words) and a rejected item sets its group's bit in grej (device, zeroed ahead of the pass).  The last block to
// finish (block counter + fence) writes the group words (1 = every item verified; a group with no items is 1) and the miss count into
// the mapped result, fences to system scope, and raises the request's completion word tail[1] = seq for the queue's thread.
__global__ void __launch_bounds__(256) k_batch_done(const uint32_t *__restrict__ items, const uint32_t *__restrict__ grp, uint32_t n_items,
                                                    uint32_t n_groups, uint32_t *grej, uint32_t *out, const uint32_t *miss_count, uint32_t *tail,
                                                    uint32_t seq, uint32_t *counter) {
  __shared__ int is_last;
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  const uint32_t gw = (n_groups + 31) / 32;
  uint32_t ok = 0;
  if (i < n_items) {
    ok = (items[i >> 5] >> (i & 31)) & 1u;
    if (!ok) {
      const uint32_t j = grp[i];
      atomicOr(grej + (j >> 5), 1u << (j & 31));
    }
  }
  const uint32_t word = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && i < n_items) out[gw + (i >> 5)] = word;
  __threadfence_system();  // this block's item words and group bits before its count
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (uint32_t w = threadIdx.x; w < gw; w += 256) out[w] = bitmap_word_ones(n_groups, w) & ~atomicOr(grej + w, 0u);
  if (threadIdx.x == 0) tail[0] = miss_count ? *(volatile const uint32_t *)miss_count : n_items;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    *counter = 0;
    __threadfence_system();
    *(volatile uint32_t *)(tail + 1) = seq;
  }
}
// all-ones bitmap over n bits (unused high bits of the last word 0)
__global__ void k_bitmap_ones(uint32_t *bm, size_t n) {
  const size_t w = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (w < (n + 31) / 32) bm[w] = bitmap_word_ones(n, w);
}
// TC::verify (consensus/src/messages.rs:307-311) and Timeout::digest (:268-275): the message of vote i is
// SHA-512(tc_round_le || high_qc_round_le)[..32] — 16 bytes of which 8 differ per vote; built and hashed here from the two
// integers (one padded block), so the host ships 8 bytes per vote instead of a digest.
__global__ void __launch_bounds__(HS_THREADS) k_tc_digests(const uint64_t *__restrict__ tc_round, const uint32_t *__restrict__ tc_idx,
                                                            const uint64_t *__restrict__ high_qc_round, size_t n, size_t n_tc, uint32_t *__restrict__ out) {
  const size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  if (i >= n) return;
  const uint32_t t = tc_idx ? tc_idx[i] : (uint32_t)i;
  const uint64_t r = t < n_tc ? tc_round[t] : 0, hq = high_qc_round[i];
  uint64_t w[16];
  // to_le_bytes() then read as big-endian message words = byte swap
  w[0] = ((uint64_t)bswap32((uint32_t)r) << 32) | bswap32((uint32_t)(r >> 32));
  w[1] = ((uint64_t)bswap32((uint32_t)hq) << 32) | bswap32((uint32_t)(hq >> 32));
  w[2] = 0x8000000000000000ULL;
#pragma unroll
  for (int j = 3; j < 15; j++) w[j] = 0;
  w[15] = 16 * 8;
  sha512_state s;
  sha512_init(s);
  sha512_compress(s, w);
  uint32_t h[16];
  sha512_output_words(s, h);
  store_digest32(out + i * 8, h);
}

// ------------------------------------------------------------------------------------------------ load generation: keygen / sign
// RFC 8032 key generation and signing of 32-byte digests (verify_core.cuh: keygen_core / sign_digest_core).  Not on the node's
// path (the reference signs one message per request on the CPU); used to synthesise benchmark and test inputs.
__global__ void __launch_bounds__(HS_THREADS) k_keygen(const uint8_t *__restrict__ seeds, size_t n, const ge_niels *__restrict__ btable,
                                                        const comb_params cp, uint8_t *__restrict__ pks) {
  __shared__ int32_t digits_s[HS_MAX_DIGITS * HS_THREADS];
  const size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  if (i >= n) return;
  uint32_t sd[8], A[8];
  load32(sd, seeds + i * 32);
  keygen_core(A, sd, btable, digits_s + threadIdx.x, HS_THREADS, cp);
  uint32_t *dst = reinterpret_cast<uint32_t *>(pks + i * 32);
#pragma unroll
  for (int j = 0; j < 8; j++) dst[j] = A[j];
}
__global__ void __launch_bounds__(HS_THREADS) k_sign_digests(const uint8_t *__restrict__ seeds, const uint8_t *__restrict__ pks,
                                                              const uint32_t *__restrict__ key_idx, const uint8_t *__restrict__ digests, size_t n,
                                                              size_t n_keys, const ge_niels *__restrict__ btable, const comb_params cp,
                                                              uint8_t *__restrict__ sig) {
  __shared__ int32_t digits_s[HS_MAX_DIGITS * HS_THREADS];
  const size_t i = (size_t)blockIdx.x * HS_THREADS + threadIdx.x;
  if (i >= n) return;
  uint32_t k = key_idx ? key_idx[i] : (uint32_t)i;
  if (k >= n_keys) k = 0;
  uint32_t sd[8], A[8], M[8], R[8], S[8];
  load32(sd, seeds + (size_t)k * 32);
  load32(A, pks + (size_t)k * 32);
  load32(M, digests + i * 32);
  sign_digest_core(R, S, sd, A, M, btable, digits_s + threadIdx.x, HS_THREADS, cp);
  uint4 *dst = reinterpret_cast<uint4 *>(sig + i * 64);
  dst[0] = make_uint4(R[0], R[1], R[2], R[3]);
  dst[1] = make_uint4(R[4], R[5], R[6], R[7]);
  dst[2] = make_uint4(S[0], S[1], S[2], S[3]);
  dst[3] = make_uint4(S[4], S[5], S[6], S[7]);
}

// ================================================================================================ host side
// ---- resource owners: the only code that creates or releases a CUDA resource, or looks up a mapped buffer's device alias
// (hs_host_alloc / hs_host_free aside: they hand pinned memory to the caller).  Every buffer, stream, event and IPC mapping of a
// context or a queue is held by one owner and released by its destructor or reset(), after whatever synchronisation its holder
// performs first.  An owner converts to its raw handle: launches, CUDA calls and
// the structs passed to kernels take that.  Owners move but never copy.
template <class H, auto Release>
class owned {
 public:
  owned() = default;
  owned(owned &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  owned &operator=(owned &&o) noexcept {
    if (this != &o) reset(std::exchange(o.h_, nullptr));
    return *this;
  }
  ~owned() { reset(); }
  void reset(H h = nullptr) {
    if (h_) Release(h_);
    h_ = h;
  }
  H get() const { return h_; }
  operator H() const { return h_; }

 private:
  H h_ = nullptr;
};
template <class T>
using dev_mem = owned<T *, cudaFree>;  // cudaMalloc
template <class T>
using pinned = owned<T *, cudaFreeHost>;  // cudaMallocHost
using stream_h = owned<cudaStream_t, cudaStreamDestroy>;
using event_h = owned<cudaEvent_t, cudaEventDestroy>;
using ipc_mapping = owned<void *, cudaIpcCloseMemHandle>;  // cudaIpcOpenMemHandle
// Mapped pinned memory (cudaHostAllocMapped): the host pointer, and its device alias, looked up once by alloc().
template <class T>
struct mapped {
  pinned<T> h;
  T *d = nullptr;
};

// Creates a resource into o through fn(&handle).  The old resource is released FIRST, so peak memory never holds both; on failure o
// stays empty.
template <class H, auto R, class Fn>
static cudaError_t acquire(owned<H, R> &o, Fn fn) {
  o.reset();
  H h = nullptr;
  const cudaError_t e = fn(&h);
  if (e == cudaSuccess) o.reset(h);
  return e;
}
template <class T>
static cudaError_t alloc(dev_mem<T> &m, size_t bytes) {
  return acquire(m, [&](T **p) { return cudaMalloc(p, bytes); });
}
template <class T>
static cudaError_t alloc(pinned<T> &m, size_t bytes) {
  return acquire(m, [&](T **p) { return cudaMallocHost(p, bytes); });
}
template <class T>
static cudaError_t alloc(mapped<T> &m, size_t bytes) {
  m.d = nullptr;
  const cudaError_t e = acquire(m.h, [&](T **p) { return cudaHostAlloc(p, bytes, cudaHostAllocMapped); });
  return e == cudaSuccess ? cudaHostGetDevicePointer(&m.d, m.h, 0) : e;
}
static cudaError_t create(stream_h &s, int priority = 0) {  // priority 0 is the default stream priority
  return acquire(s, [&](cudaStream_t *p) { return cudaStreamCreateWithPriority(p, cudaStreamNonBlocking, priority); });
}
static cudaError_t create(event_h &ev, unsigned flags = cudaEventDisableTiming) {
  return acquire(ev, [&](cudaEvent_t *p) { return cudaEventCreateWithFlags(p, flags); });
}
static cudaError_t ipc_open(ipc_mapping &m, cudaIpcMemHandle_t h) {
  return acquire(m, [&](void **p) { return cudaIpcOpenMemHandle(p, h, cudaIpcMemLazyEnablePeerAccess); });
}
// ---- end of resource owners

struct dev_buf {  // grow-only device scratch (ensure())
  dev_mem<void> p;
  size_t cap = 0;
};
// The committee's or the key cache's tables: keys, key flags, the key hash table and the per-key comb tables.  Built whole in a local
// and moved in, so a failed registration or key-cache allocation leaves none of them.
struct key_store {
  dev_mem<uint8_t> pks;
  dev_mem<uint8_t> key_flags;
  dev_mem<ge_niels> atables;
  dev_mem<uint32_t> slots;
};
// A key store of n_slots slots with tables at window wa and a hash table of hash_slots entries, empty on `stream`: flags 0, hash slots
// 0xff (HS_NO_KEY).  Moved into `out` only when every allocation succeeded.
static cudaError_t make_key_store(key_store &out, size_t n_slots, size_t hash_slots, int wa, cudaStream_t stream) {
  key_store K;
  cudaError_t e = alloc(K.pks, n_slots * 32);
  if (e == cudaSuccess) e = alloc(K.key_flags, n_slots);
  if (e == cudaSuccess) e = alloc(K.slots, hash_slots * 4);
  if (e == cudaSuccess) e = alloc(K.atables, n_slots * comb_table_entries(wa) * sizeof(ge_niels));
  if (e == cudaSuccess) e = cudaMemsetAsync(K.key_flags, 0, n_slots, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(K.slots, 0xff, hash_slots * 4, stream);
  if (e == cudaSuccess) out = std::move(K);
  return e;
}
// Key-cache learning: the unknown keys of a pass and their count, their pinned host copies, and the events.  Allocated whole on first use.
struct learn_bufs {
  dev_mem<uint8_t> keys;
  dev_mem<uint32_t> n;
  pinned<uint8_t> h_keys;
  pinned<uint32_t> h_n;
  pinned<uint32_t> h_miss_total;  // total misses of the pass whose keys are parked
  event_h ev;
  event_h ev_tables;  // recorded after the latest table build of the key cache; every pass waits for it (any stream)
};
// hs_table_audit: its private lowest-priority stream, the event recorded after its kernels, and its scratch.  Created on first use.
struct audit_state {
  stream_h stream;
  event_h done;
  dev_buf scratch;
  dev_buf stage;  // hs_table_mend's staging: HS_BUILD_BLOCK + 1 entries per thread of one k_mend_windows launch
};
// A ring of slots that k_verify_small, k_verify_bulk, k_queue_generic and k_queue_digests work over (slot = position & mask): the
// latency path's (one request in slot 0), a verify queue's and the self-test's.
struct ring_bufs {
  mapped<small_rec> recs;      // sig | msg | vidx | req | req_n per record
  mapped<uint8_t> flags;       // verdict flags per record
  mapped<uint32_t> done;       // completion word per request slot (= launch sequence number)
  dev_mem<uint32_t> counters;  // records finished per request slot
};
// Allocates r for cap slots.  When it returns, the completion words and the counters are 0.
static cudaError_t make_ring(ring_bufs &r, uint32_t cap, cudaStream_t stream) {
  cudaError_t e = alloc(r.recs, (size_t)cap * sizeof(small_rec));
  if (e == cudaSuccess) e = alloc(r.flags, cap);
  if (e == cudaSuccess) e = alloc(r.done, (size_t)cap * 4);
  if (e == cudaSuccess) e = alloc(r.counters, (size_t)cap * 4);
  if (e == cudaSuccess) e = cudaMemsetAsync(r.counters, 0, (size_t)cap * 4, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);  // the ring's kernels may run on other streams
  if (e == cudaSuccess) memset(r.done.h, 0, (size_t)cap * 4);
  return e;
}
// Multi-GPU peer routing: this rank's result buffer (cudaMalloc'd: [2][total_words][HS_MAX_PEERS flags][timeout flag, block counter])
// and the mappings of the other ranks' buffers.
struct peer_bufs {
  dev_mem<uint32_t> own;
  ipc_mapping mapped[HS_MAX_PEERS];
};
enum : uint8_t { SLOT_LIVE = 1, SLOT_REPAIR = 2, SLOT_STAGED = 3 };  // hs_ctx::h_key_live values of a slot in use
// A staged committee change (hs_committee_stage): its slots are SLOT_STAGED in h_key_live, out of service, until the commit.
struct committee_stage {
  bool busy = false;            // the stage holds slots: being built, or built and proved
  bool ready = false;           // built and proved: hs_committee_commit applies it
  std::vector<uint32_t> fresh;  // the slots it took, lowest free first, then spares (those past n_keys are consecutive from it)
  std::vector<uint8_t> keys;    // their key bytes (32 each)
  std::vector<uint8_t> flags;   // their proved flag bytes
  std::vector<uint32_t> remove; // the slots the commit takes out of service
  // A staged registration (hs_committee_stage_register): `whole`, with no slot above.  keys and flags hold its N keys and their proved
  // flag bytes; `store` is the new key store beside the live one (moved in here only once proved), with its index, slots and window.
  bool whole = false;
  key_store store;
  key_index index;
  size_t capacity = 0;
  int wa = 0;
};
// The engine-owned scrub (hs_scrub_start): its thread, the map it audits against and where its pass stands.  `m` guards all but `th`
// (hs_scrub_start / hs_scrub_stop, under hs_ctx::scrub_life) and the counters (read at any time).  Lock order: m, audit_mu, mu.
// hs_table_mend_stats: calls, windows recomputed, entries rewritten, windows left, slots left to repair, cache flushes
enum { MEND_CALLS, MEND_WINDOWS, MEND_REWRITTEN, MEND_WINDOWS_LEFT, MEND_SLOTS_LEFT, MEND_FLUSHES, MEND_NSTATS };
enum { SCRUB_PASSES, SCRUB_SLOTS, SCRUB_BASE, SCRUB_TICKS, SCRUB_FINDINGS, SCRUB_REPAIRED, SCRUB_FAILED, SCRUB_PAUSED, SCRUB_NSTATS };
struct scrub_state {
  std::thread th;
  std::mutex m;
  std::condition_variable cv;
  bool stop = false;
  int rc = 0;                       // the error that ended the thread early (returned by hs_scrub_stop)
  // the map: the caller's (has_pks / has_live) or the engine's own, for the slot map of generation map_gen
  std::vector<uint8_t> pks;
  std::vector<uint32_t> live;
  bool has_pks = false, has_live = false;
  size_t n_slots = 0;
  uint64_t map_gen = 0;
  uint32_t period_us = 0, slots_per_tick = 0, base_per_tick = 0;
  bool mend = false;                // hs_scrub_mend: a tick whose findings can all be mended mends them instead of repairing
  hs_scrub_cb *cb = nullptr;
  void *user = nullptr;
  size_t next_slot = 0;             // the pass: the slots before next_slot and the base entries before next_base are audited
  uint64_t next_base = 0;
  // hs_scrub_sig_cache: the queue whose signature cache each tick also audits, sig_per_tick buckets from sig_next on, in the table of
  // generation sig_gen (a new table starts at bucket 0)
  hs_queue *sig_q = nullptr;
  uint32_t sig_per_tick = 0, sig_gen = 0;
  size_t sig_next = 0;
  std::atomic<uint64_t> stats[SCRUB_NSTATS] = {};
};
struct hs_ctx {
  int device = 0;
  unsigned n_sms = 0;                // multiprocessors of `device` (sizes the grid of the side pass)
  stream_h stream, stream2, stream_side;
  event_h ev[2], ev_done[2], ev_side[2];
  // recorded after the last enqueue of every `_dev` verify pass on a caller's stream: the host-pointer calls reuse the same scratch on
  // `stream`, which waits for it before its first enqueue (h2d_stage::upload on `stream`, hs_verify_msgs)
  event_h ev_dev_pass;
  dev_mem<ge_niels> d_btable;
  comb_params cp{};
  size_t a_table_entries = 0;
  int wa_forced = 0;
  // committee
  size_t n_keys = 0;
  key_store keys;
  // grow-only device scratch
  dev_buf in[2], digest[2], xyz, meta, vidx, miss, out;
  dev_buf group_digests;  // hs_verify_groups_dev: Digests of the pass's preimages (read by the main kernels only, so one set serves deferred mode)
  dev_buf explain_sel;    // hs_explain_groups_dev: block offsets, then the selected item list (not the verify scratch: host calls never wait for it)
  dev_mem<uint32_t> d_miss_count;
  // key cache: tables for keys that were never registered but keep showing up (learned between calls)
  bool explicit_committee = false;   // hs_committee_register was called with keys: the set is fixed, nothing is learned
  bool cache_wanted = true, cache_enabled = true;
  size_t cache_cap = 4096;           // keys
  std::vector<uint8_t> h_pks;        // host mirrors of keys.pks / keys.slots (key cache and hs_committee_update)
  key_index h_index;
  std::vector<uint8_t> h_key_live;   // explicit committee: SLOT_LIVE, SLOT_REPAIR (live, out of service during hs_table_repair), SLOT_STAGED
                                     // (taken by a stage, past n_keys for a spare) or 0 = removed (free for reuse)
  committee_stage stage;             // guarded by mu
  size_t table_budget = 0;           // bytes the per-key tables may use (0 = ~62 % of the device)
  size_t key_capacity = 0;           // explicit committee: table slots allocated (>= n_keys; spare slots serve hs_committee_update)
  learn_bufs learn;
  bool learn_pending = false;
  bool cache_full = false;           // no free slot: only the miss RATE is watched (a mostly-missing full cache is reset)
  uint64_t calls_since_reset = HS_CACHE_RESET_MIN_CALLS;
  size_t learn_records = 0;          // records of the pass whose misses are parked in learn.h_*
  // key-table generation: bumped (under mu) by every path that frees or rewrites the per-key tables, key bytes, flags or hash table, so
  // an audit that ran across such a change reports nothing.  Those paths first wait for audit.done (or synchronise the device).
  uint64_t key_gen = 0;
  // slot-map generation: bumped with key_gen by registration, hs_committee_update, hs_committee_commit and the key cache's changes,
  // i.e. whenever hs_key_slots or a slot's key or liveness changes; a repair restores the map and leaves it alone.
  uint64_t map_gen = 0;
  std::mutex audit_mu;               // one hs_table_audit at a time: it owns `audit` for the whole call, `mu` only briefly
  audit_state audit;
  std::atomic<uint64_t> mend_stats[MEND_NSTATS] = {};  // hs_table_mend_stats (the scrub's mends included)
  std::mutex scrub_life;             // hs_scrub_start / hs_scrub_stop: starting and joining the scrub's thread
  scrub_state scrub;
  // multi-GPU peer routing
  peer_route peers{};
  int peer_rank = 0;
  size_t peer_total_words = 0;
  peer_bufs peer;
  bool peer_armed = false;
  uint32_t peer_epoch = 0;
  // latency path
  ring_bufs small;  // HS_SMALL_MAX slots
  uint32_t small_seq = 0;
  bool small_enabled = true;
  // deferred-results mode (hs_set_deferred): the latency-bound tail of a `_dev` verify pass (finish kernel, peer exchange, per-QC AND)
  // runs on an internal stream so that it overlaps the main kernel of the NEXT pass; two scratch sets alternate
  bool deferred = false;
  stream_h stream_tail;
  event_h ev_main_done, ev_tail[2], ev_results;
  dev_buf xyz2, meta2;
  int flip = 0;
  // optional timing of the dominant kernel alone (bench.py's roofline): events around k_verify_main<committee>
  bool profile_main = false;
  event_h ev_prof[2];
  std::atomic<uint64_t> launches{0};
  std::mutex mu;
  std::mutex err_mu;                  // guards err only: fail() is also reached from argument checks taken before `mu`
  std::string err = "ok";
  std::mutex queues_mu;               // guards queues only (hs_ctx_destroy tears them down without holding `mu`)
  std::vector<hs_queue *> queues;     // verify queues attached to this context
  // hs_queue_sig_share (under mu): the queue whose signature cache the host-pointer verify calls share; the table of the call in
  // progress (b == nullptr: it does not share) and its shared passes; their scratch, device counters and mapped copy of the counts
  hs_queue *share_q = nullptr;
  sig_cache_dev share_sc{};
  uint32_t share_passes = 0;
  dev_buf share_list, share_fl;
  dev_mem<uint32_t> share_ctr;  // HS_SIG_CTRS counts, then the miss list's count
  mapped<uint32_t> share_h;     // HS_SIG_CTRS
};
// The context holds per-key tables: a registered committee's or learned keys'.  Registration, hs_committee_update and learn_process
// raise n_keys only once `keys` is in place, and cache_release clears both, so n_keys > 0 alone implies the second term.
static bool has_key_tables(const hs_ctx *c) { return c->n_keys > 0 && c->keys.atables; }
// A committee is registered: its key set is fixed and nothing is learned.  explicit_committee is set only once the store is in place.
static bool committee_registered(const hs_ctx *c) { return c->explicit_committee && has_key_tables(c); }

static int fail(hs_ctx *c, int code, const char *what, cudaError_t e = cudaSuccess) {
  if (c) {
    std::lock_guard<std::mutex> g(c->err_mu);
    c->err = what;
    if (e != cudaSuccess) {
      c->err += ": ";
      c->err += cudaGetErrorString(e);
    }
  }
  return code;
}
#define HS_CUDA(c, call)                                               \
  do {                                                                 \
    cudaError_t e__ = (call);                                          \
    if (e__ != cudaSuccess) return fail((c), HS_ERR_CUDA, #call, e__); \
  } while (0)
#define HS_TRY(expr)          \
  do {                        \
    int rc__ = (expr);        \
    if (rc__) return rc__;    \
  } while (0)

static int ensure(hs_ctx *c, dev_buf &b, size_t need) {
  if (need <= b.cap) return HS_OK;
  if (b.p) cudaDeviceSynchronize();  // the old block may still be in flight on another stream
  b.cap = 0;
  size_t want = need + need / 4 + 4096;
  cudaError_t e = alloc(b.p, want);  // frees the old block first
  if (e != cudaSuccess) return fail(c, HS_ERR_NOMEM, "cudaMalloc scratch", e);
  b.cap = want;
  return HS_OK;
}
static inline unsigned blocks_for(size_t n, unsigned per = HS_THREADS) { return (unsigned)((n + per - 1) / per); }

// A host entry point's inputs, staged into one grow-only device buffer.  add() declares the sections in order: each starts 16-byte
// aligned and is followed by `slack` spare bytes; src == nullptr reserves the bytes without copying them.  upload() ensures the
// buffer and copies every non-empty section that has a source.  ptr() is valid only after upload(), since ensure() may move the
// buffer, and is a valid address even for a section of 0 bytes.
struct h2d_stage {
  struct section {
    const void *src;
    size_t off, bytes;
  };
  std::array<section, 8> sec;  // at() in add() throws on a ninth section
  size_t n = 0, total = 0;
  uint8_t *base = nullptr;
  size_t add(const void *src, size_t bytes, size_t slack = 0) {
    const size_t off = (total + 15) & ~(size_t)15;
    sec.at(n) = {src, off, bytes};
    total = off + bytes + slack;
    return n++;
  }
  int upload(hs_ctx *c, dev_buf &buf, cudaStream_t stream) {
    // The host-pointer entry points stage on the context's stream and then run passes over the verify scratch, which a `_dev` pass on
    // the caller's stream may still read: they wait for it.  The self-test, the audit, the scrub and slot builds stage on streams of
    // their own for work over scratch of their own, and do not.
    if (stream == c->stream) HS_CUDA(c, cudaStreamWaitEvent(stream, c->ev_dev_pass, 0));
    HS_TRY(ensure(c, buf, total));
    base = (uint8_t *)buf.p.get();
    for (size_t k = 0; k < n; k++)
      if (sec[k].src && sec[k].bytes) HS_CUDA(c, cudaMemcpyAsync(base + sec[k].off, sec[k].src, sec[k].bytes, cudaMemcpyHostToDevice, stream));
    return HS_OK;
  }
  uint8_t *ptr(size_t k) const { return base + sec[k].off; }
};
// A host entry point's results: every copy with a destination, on the context's stream, then one wait for the stream.
struct d2h_copy {
  void *dst;  // nullable: an output the caller did not ask for
  const void *src;
  size_t bytes;
};
static int readback(hs_ctx *c, std::initializer_list<d2h_copy> copies) {
  for (const d2h_copy &r : copies)
    if (r.dst) HS_CUDA(c, cudaMemcpyAsync(r.dst, r.src, r.bytes, cudaMemcpyDeviceToHost, c->stream));
  HS_CUDA(c, cudaStreamSynchronize(c->stream));
  return HS_OK;
}
// The words of an all-ones bitmap over n bits: the initial group words of a certificate pass, kept off the caller's buffer so that a
// call that fails leaves it unwritten.
static std::vector<uint32_t> bitmap_ones(size_t n) {
  std::vector<uint32_t> bm((n + 31) / 32);
  for (size_t w = 0; w < bm.size(); w++) bm[w] = bitmap_word_ones(n, w);
  return bm;
}
// Clears bit j of d_groups when an item with d_group_idx == j is rejected, over an item bitmap of n_items bits.
static int launch_qc_and(hs_ctx *c, const uint32_t *d_items, const uint32_t *d_group_idx, size_t n_items, size_t n_groups, uint32_t *d_groups,
                         cudaStream_t stream) {
  k_qc_and<<<blocks_for(n_items, 256), 256, 0, stream>>>(d_items, d_group_idx, n_items, n_groups, d_groups);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}


// k_build_comb over n_points points: slots 0 .. n_points - 1 of d_encs / tables, or with d_slots the listed slots (flags by list position).
static int launch_build(hs_ctx *c, const uint8_t *d_encs, const uint32_t *d_slots, size_t n_points, int negate, int W, int n_windows,
                        ge_niels *tables, uint8_t *flags, cudaStream_t stream) {
  size_t threads = n_points * (size_t)n_windows * ((1u << (W - 1)) / HS_BUILD_BLOCK);
  k_build_comb<<<blocks_for(threads), HS_THREADS, 0, stream>>>(d_encs, d_slots, n_points, negate, W, n_windows, tables, flags);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}

static void set_window(comb_params &cp, bool a, int w) {
  if (a) {
    cp.wa = w;
    cp.na = sc_ndigits_rt(w);
    sc_bias_rt(cp.bias_a, w);
  } else {
    cp.wb = w;
    cp.nb = sc_ndigits_rt(w);
    sc_bias_rt(cp.bias_b, w);
  }
}

// ---- key cache -----------------------------------------------------------------------------------------------------
// Before a key-cache path rewrites tables, key bytes or the hash table on `stream`: an audit's kernels in flight finish first.
static int audit_fence(hs_ctx *c, cudaStream_t stream) {
  c->key_gen++;
  c->map_gen++;
  if (c->audit.done) HS_CUDA(c, cudaStreamWaitEvent(stream, c->audit.done, 0));
  return HS_OK;
}
static void cache_release(hs_ctx *c) {  // callers have synchronised the device
  c->key_gen++;
  c->map_gen++;
  c->keys = {};
  c->n_keys = 0;
  c->h_pks.clear();
  c->h_index = {};
  c->h_key_live.clear();
  c->stage = {};  // a registration discards a pending stage: its slots went with the store
  c->key_capacity = 0;
}
// lazily allocate the store for cache_cap learned keys (14-bit windows: 14 MB per key, narrower if memory is short)
static int cache_allocate(hs_ctx *c, cudaStream_t stream) {
  size_t free_b = 0, total_b = 0;
  HS_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  size_t lim = free_b / 2;
  if (c->table_budget && c->table_budget < lim) lim = c->table_budget;
  int wa = 8;
  for (int w : {14, 12, 10, 8}) {
    if (c->wa_forced && w != c->wa_forced && w != 8) continue;
    wa = w;
    if (c->cache_cap * comb_table_entries(w) * sizeof(ge_niels) <= lim) break;
  }
  if (c->cache_cap * comb_table_entries(wa) * sizeof(ge_niels) > lim || sc_ndigits_rt(wa) + c->cp.nb > HS_MAX_DIGITS) {
    c->cache_enabled = false;  // not enough memory: stay on the generic path
    return HS_OK;
  }
  set_window(c->cp, true, wa);
  c->a_table_entries = comb_table_entries(wa);
  HS_CUDA(c, make_key_store(c->keys, c->cache_cap, key_index::capacity_for(c->cache_cap), wa, stream));
  c->key_gen++;  // nothing to wait for: the store had no tables, so no audit reads it
  c->map_gen++;
  c->h_index.reset(c->cache_cap);
  c->h_pks.clear();
  return HS_OK;
}
// Called at the start of a verify pass: if the previous pass left unknown keys behind (already copied to pinned host memory),
// dedupe them, append the new ones to the store and build their comb tables on `stream` before this pass's lookup runs.
static int learn_process(hs_ctx *c, cudaStream_t stream) {
  if (!c->learn_pending) return HS_OK;
  if (cudaEventQuery(c->learn.ev) != cudaSuccess) return HS_OK;  // copy still in flight: try again on the next call
  c->learn_pending = false;
  c->calls_since_reset++;
  if (!c->cache_enabled || c->explicit_committee) return HS_OK;
  if (c->cache_full) {
    // Full cache that no longer matches the traffic (e.g. the validator set rotated): more than half of the last pass missed.
    // Start over — the next passes relearn the keys that are actually in use.  (No per-key eviction; see DESIGN.md §8.)
    if (c->learn_records >= 64 && (size_t)*c->learn.h_miss_total * 2 > c->learn_records && c->calls_since_reset >= HS_CACHE_RESET_MIN_CALLS) {
      c->calls_since_reset = 0;
      HS_TRY(audit_fence(c, stream));
      c->n_keys = 0;
      c->h_pks.clear();
      c->h_index.clear();
      HS_CUDA(c, cudaMemsetAsync(c->keys.slots, 0xff, c->h_index.slots.size() * 4, stream));
      c->cache_full = false;
    }
    return HS_OK;
  }
  const uint32_t got = *c->learn.h_n < HS_LEARN_MAX ? *c->learn.h_n : HS_LEARN_MAX;
  if (got == 0) return HS_OK;
  if (!c->keys.atables) {
    HS_TRY(cache_allocate(c, stream));
    if (!c->cache_enabled) return HS_OK;
  }
  const size_t old_n = c->n_keys;
  size_t n_new = 0;
  for (uint32_t t = 0; t < got && old_n + n_new < c->cache_cap && n_new < HS_LEARN_PER_CALL; t++) {
    const uint8_t *key = c->learn.h_keys + 32 * (size_t)t;
    c->h_pks.insert(c->h_pks.end(), key, key + 32);
    if (c->h_index.insert_absent(c->h_pks.data(), (uint32_t)(old_n + n_new))) n_new++;
    else c->h_pks.resize(32 * (old_n + n_new));  // already learned
  }
  if (n_new == 0) return HS_OK;
  HS_TRY(audit_fence(c, stream));
  HS_CUDA(c, cudaMemcpyAsync(c->keys.pks + old_n * 32, c->h_pks.data() + old_n * 32, n_new * 32, cudaMemcpyHostToDevice, stream));
  HS_CUDA(c, cudaMemcpyAsync(c->keys.slots, c->h_index.slots.data(), c->h_index.slots.size() * 4, cudaMemcpyHostToDevice, stream));
  HS_TRY(launch_build(c, c->keys.pks + old_n * 32, nullptr, n_new, 1, c->cp.wa, c->cp.na, c->keys.atables + old_n * c->a_table_entries,
                      c->keys.key_flags + old_n, stream));
  // (no synchronisation: copies from pageable memory return once the source is staged, so the host vectors may change afterwards)
  HS_CUDA(c, cudaEventRecord(c->learn.ev_tables, stream));  // passes on OTHER streams (host entry points vs a _dev caller's stream) wait for the build
  c->n_keys = old_n + n_new;
  if (c->n_keys >= c->cache_cap) c->cache_full = true;  // no free slot: unknown keys stay on the generic path until a reset
  return HS_OK;
}
// After the lookup of a pass: park the unknown keys for learn_process().
static int learn_collect(hs_ctx *c, const in_layout &L, size_t n, bool have_lookup, cudaStream_t stream) {
  if (!c->cache_enabled || c->explicit_committee || c->learn_pending || !L.pk) return HS_OK;
  if (!c->learn.keys) {  // first use: every buffer, or none
    learn_bufs B;
    HS_CUDA(c, alloc(B.keys, (size_t)HS_LEARN_MAX * 32));
    HS_CUDA(c, alloc(B.n, 4));
    HS_CUDA(c, alloc(B.h_keys, (size_t)HS_LEARN_MAX * 32));
    HS_CUDA(c, alloc(B.h_n, 4));
    HS_CUDA(c, alloc(B.h_miss_total, 4));
    HS_CUDA(c, create(B.ev));
    HS_CUDA(c, create(B.ev_tables));
    c->learn = std::move(B);
  }
  learn_bufs &B = c->learn;
  c->learn_records = n;
  if (c->cache_full) {  // only watch the miss rate
    if (!have_lookup) return HS_OK;
    HS_CUDA(c, cudaMemcpyAsync(B.h_miss_total, c->d_miss_count, 4, cudaMemcpyDeviceToHost, stream));
    HS_CUDA(c, cudaEventRecord(B.ev, stream));
    c->learn_pending = true;
    return HS_OK;
  }
  k_gather_keys<<<blocks_for(HS_LEARN_MAX, 256), 256, 0, stream>>>(L, n, have_lookup ? (const uint32_t *)c->miss.p.get() : nullptr,
                                                                     have_lookup ? c->d_miss_count.get() : nullptr, HS_LEARN_MAX, B.keys, B.n);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  HS_CUDA(c, cudaMemcpyAsync(B.h_n, B.n, 4, cudaMemcpyDeviceToHost, stream));
  HS_CUDA(c, cudaMemcpyAsync(B.h_keys, B.keys, (size_t)HS_LEARN_MAX * 32, cudaMemcpyDeviceToHost, stream));
  HS_CUDA(c, cudaEventRecord(B.ev, stream));
  c->learn_pending = true;
  return HS_OK;
}

// Scratch and streams of one verify pass's main phase: the context's for run_verify, a verify queue's batch lane for its passes.
struct pass_scratch {
  fe *xyz;
  uint8_t *meta;
  uint32_t *vidx, *miss, *miss_count;  // k_key_lookup's outputs (table path with key bytes)
  cudaStream_t side;                   // the generic pass over the lookup's misses
  cudaEvent_t ev_side[2];
  const event_h *prof;                 // nullable: events around k_verify_main<committee>
};
// The per-key tables a verify pass reads and the windows they were built at: the context's (registered committee or key cache), or
// the scratch set of hs_self_test.  The base-point table is always the context's.
struct pass_tables {
  committee_tables C;
  key_table T;
  comb_params cp;
};
// The view of key store S whose first n_keys slots hold tables of `entries` entries at window cp.wa, found through `index`.
static pass_tables store_tables(const key_store &S, const key_index &index, size_t n_keys, size_t entries, const comb_params &cp) {
  return pass_tables{{S.pks, S.key_flags, (uint32_t)n_keys, S.atables, entries}, {S.slots, index.mask, S.pks, (uint32_t)n_keys}, cp};
}
static pass_tables ctx_tables(const hs_ctx *c) { return store_tables(c->keys, c->h_index, c->n_keys, c->a_table_entries, c->cp); }
// A pass that shares a queue's signature cache (hs_queue_sig_share): the table, the pass's device counters (sc.ctr, HS_SIG_CTRS words,
// then the miss list's count), the miss list, every record's flag byte, and the mapped words its counts are copied to at the end.
struct share_pass {
  sig_cache_dev sc;
  uint32_t *list;
  uint8_t *fl;
  uint32_t *h_ctr;
};
// A pass on `stream` reads the key cache's tables only after their latest build, which learn_process may have enqueued on another stream.
static int wait_key_cache_build(hs_ctx *c, cudaStream_t stream) {
  if (c->learn.ev_tables && !c->explicit_committee) HS_CUDA(c, cudaStreamWaitEvent(stream, c->learn.ev_tables, 0));
  return HS_OK;
}
// The main phase on `stream`: with committee tables, [k_key_lookup, then k_verify_main<false> over the misses on S.side] beside
// k_verify_main<true>; without, k_verify_main<false> over every record.  after_lookup(have_lookup) runs where run_verify collects
// keys for the key cache.  L.vidx is set to the lookup's indices when it runs.  sh (nullable, committee passes only): k_sig_probe
// decides the records the cache holds and k_verify_main<true> runs over the list of the others.
template <class AfterLookup>
static int launch_main(hs_ctx *c, in_layout &L, size_t n, bool committee, bool indexed, const pass_tables &K, const pass_scratch &S,
                       cudaStream_t stream, AfterLookup after_lookup, const share_pass *sh = nullptr) {
  main_out O{S.xyz, S.meta, 0};
  const committee_tables &C = K.C;
  if (committee) {
    if (!indexed) {
      HS_CUDA(c, cudaMemsetAsync(S.miss_count, 0, 4, stream));
      k_key_lookup<<<blocks_for(n, 256), 256, 0, stream>>>(L, n, K.T, S.vidx, S.miss, S.miss_count);
      c->launches++;
      HS_CUDA(c, cudaGetLastError());
      L.vidx = S.vidx;
      O.side_pass = 1;
      HS_TRY(after_lookup(true));
      // Records whose key is not registered take the generic path over the compacted list.  One generic verify has a
      // ~0.8 ms single-warp latency, so the pass runs on the high-priority side stream CONCURRENTLY with the committee
      // pass (disjoint outputs); its length stays on the device (no host round trip).
      HS_CUDA(c, cudaEventRecord(S.ev_side[0], stream));
      HS_CUDA(c, cudaStreamWaitEvent(S.side, S.ev_side[0], 0));
      unsigned grid = blocks_for(n, 32);
      if (grid > c->n_sms * 8u) grid = c->n_sms * 8u;
      k_verify_main<false><<<grid, 32, 0, S.side>>>(L, 0, S.miss_count, S.miss, c->d_btable, C, O, K.cp);
      c->launches++;
      HS_CUDA(c, cudaGetLastError());
      HS_CUDA(c, cudaEventRecord(S.ev_side[1], S.side));
    }
    const uint32_t *n_ptr = nullptr, *list = nullptr;
    if (sh) {
      uint32_t *list_n = sh->sc.ctr + HS_SIG_CTRS;
      HS_CUDA(c, cudaMemsetAsync(sh->sc.ctr, 0, 4 * (HS_SIG_CTRS + 1), stream));
      k_sig_probe<<<blocks_for(n, 256), 256, 0, stream>>>(L, n, C, sh->sc, indexed ? 0 : 1, S.xyz, S.meta, sh->list, list_n);
      c->launches++;
      HS_CUDA(c, cudaGetLastError());
      n_ptr = list_n;
      list = sh->list;
    }
    if (S.prof) HS_CUDA(c, cudaEventRecord(S.prof[0], stream));
    k_verify_main<true><<<blocks_for(n), HS_THREADS, 0, stream>>>(L, n, n_ptr, list, c->d_btable, C, O, K.cp);
    if (S.prof) HS_CUDA(c, cudaEventRecord(S.prof[1], stream));
    c->launches++;
    HS_CUDA(c, cudaGetLastError());
    if (!indexed) HS_CUDA(c, cudaStreamWaitEvent(stream, S.ev_side[1], 0));
  } else {
    HS_TRY(after_lookup(false));
    k_verify_main<false><<<blocks_for(n), HS_THREADS, 0, stream>>>(L, n, nullptr, nullptr, c->d_btable, C, O, K.cp);
    c->launches++;
    HS_CUDA(c, cudaGetLastError());
  }
  return HS_OK;
}
// Threads of k_verify_finish own `fin_group` records each; launched on `stream`.  d_item_mode (device, nullable): record i is judged
// by its own mode byte (k_verify_finish_modes) instead of `mode`.  sh (nullable): the pass shares a signature cache, so the cached
// kernels run and write every record's flag byte to sh->fl.
static int launch_finish(hs_ctx *c, const in_layout &L, size_t n, const fe *xyz, const uint8_t *meta, uint32_t mode, const uint8_t *d_item_mode,
                         uint32_t *d_bitmap, const peer_route &P, int fin_group, cudaStream_t stream, const share_pass *sh = nullptr) {
  const size_t fin_threads = (n + fin_group - 1) / fin_group;
  if (sh && d_item_mode)
    k_verify_finish_modes_cached<<<blocks_for(fin_threads), HS_THREADS, 0, stream>>>(L, n, xyz, meta, d_item_mode, d_bitmap, P, fin_group, sh->fl);
  else if (sh)
    k_verify_finish_cached<<<blocks_for(fin_threads), HS_THREADS, 0, stream>>>(L, n, xyz, meta, mode, d_bitmap, P, fin_group, sh->fl);
  else if (d_item_mode)
    k_verify_finish_modes<<<blocks_for(fin_threads), HS_THREADS, 0, stream>>>(L, n, xyz, meta, d_item_mode, d_bitmap, P, fin_group);
  else
    k_verify_finish<<<blocks_for(fin_threads), HS_THREADS, 0, stream>>>(L, n, xyz, meta, mode, d_bitmap, P, fin_group);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
// The end of a shared pass, after its finish kernel on `stream`: k_sig_fill, then the pass's counts to sh.h_ctr.
static int launch_sig_fill(hs_ctx *c, const in_layout &L, size_t n, const committee_tables &C, const share_pass &sh, const uint8_t *meta,
                           uint32_t mode, const uint8_t *d_item_mode, cudaStream_t stream) {
  k_sig_fill<<<blocks_for(n, 256), 256, 0, stream>>>(L, n, C, sh.sc, meta, sh.fl, mode, d_item_mode);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  HS_CUDA(c, cudaMemcpyAsync(sh.h_ctr, sh.sc.ctr, 4 * HS_SIG_CTRS, cudaMemcpyDeviceToHost, stream));
  return HS_OK;
}

// Runs lookup (optional) -> main (committee and/or generic) -> finish on `stream` for a device-resident layout.
// use_lookup: L.pk is valid and a committee is registered -> resolve indices on the device.
// d_item_mode (device, nullable): per-record verdict modes in place of `mode`; read by the finish kernel (on the tail stream when deferred).
static int run_verify(hs_ctx *c, in_layout L, size_t n, uint32_t mode, uint32_t *d_bitmap, cudaStream_t stream, bool indexed,
                      const uint8_t *d_item_mode = nullptr) {
  if (n == 0) {
    if (c->peer_armed) {  // an empty shard still owes its peers the epoch flag
      c->peer_armed = false;
      k_peer_sync_only<<<1, HS_MAX_PEERS, 0, stream>>>(c->peers);
      c->launches++;
      HS_CUDA(c, cudaGetLastError());
    }
    return HS_OK;
  }
  if (indexed && !committee_registered(c)) return fail(c, HS_ERR_ARG, "committee-indexed verify without a registered committee");
  if (!indexed) HS_TRY(learn_process(c, stream));
  HS_TRY(wait_key_cache_build(c, stream));
  const bool defer = c->deferred && stream != c->stream;  // host-pointer entry points (internal stream) always complete in stream order
  dev_buf &XYZ = (defer && c->flip) ? c->xyz2 : c->xyz, &META = (defer && c->flip) ? c->meta2 : c->meta;
  const int set = defer ? c->flip : 0;
  if (defer) {
    c->flip ^= 1;
    HS_CUDA(c, cudaStreamWaitEvent(stream, c->ev_tail[set], 0));  // the finish kernel that last read this scratch set is done
  }
  HS_TRY(ensure(c, XYZ, n * 3 * sizeof(fe)));
  HS_TRY(ensure(c, META, n));
  const bool committee = has_key_tables(c) && (indexed || L.pk);
  if (!committee && !L.pk) return fail(c, HS_ERR_ARG, "verify without keys");
  if (committee && !indexed) {
    HS_TRY(ensure(c, c->vidx, n * 4));
    HS_TRY(ensure(c, c->miss, n * 4));
  }
  const pass_scratch S{(fe *)XYZ.p.get(), (uint8_t *)META.p.get(), (uint32_t *)c->vidx.p.get(), (uint32_t *)c->miss.p.get(), c->d_miss_count, c->stream_side,
                       {c->ev_side[0], c->ev_side[1]}, c->profile_main ? c->ev_prof : nullptr};
  // a host-pointer call that shares a signature cache (share_call), over 32-byte messages (so on the context's stream, never deferred)
  const bool share = c->share_sc.b && committee && stream == c->stream && !L.off && L.fixed_len == 32;
  share_pass SP{};
  if (share) {
    HS_TRY(ensure(c, c->share_list, n * 4));
    HS_TRY(ensure(c, c->share_fl, n));
    SP = share_pass{c->share_sc, (uint32_t *)c->share_list.p.get(), (uint8_t *)c->share_fl.p.get(), c->share_h.h};
  }
  HS_TRY(launch_main(c, L, n, committee, indexed, ctx_tables(c), S, stream,
                     [&](bool have_lookup) { return learn_collect(c, L, n, have_lookup, stream); }, share ? &SP : nullptr));
  // small batches: small groups, so that enough blocks exist to hide each block's serial inversion; when the tail overlaps the next pass
  // (deferred mode) latency is hidden anyway and the 16-record group costs the fewest inversions
  const int fin_group = (defer || n >= (1u << 19)) ? 16 : (n >= (1u << 18) ? 8 : 4);
  peer_route P{};
  if (c->peer_armed) {
    P = c->peers;
    c->peer_armed = false;
  }
  cudaStream_t fin_stream = stream;
  if (defer) {  // tail on the internal stream: the caller's stream is free for the next pass's digest / main kernels
    HS_CUDA(c, cudaEventRecord(c->ev_main_done, stream));
    HS_CUDA(c, cudaStreamWaitEvent(c->stream_tail, c->ev_main_done, 0));
    fin_stream = c->stream_tail;
  }
  HS_TRY(launch_finish(c, L, n, (const fe *)XYZ.p.get(), (const uint8_t *)META.p.get(), mode, d_item_mode, d_bitmap, P, fin_group, fin_stream,
                       share ? &SP : nullptr));
  if (share) {
    HS_TRY(launch_sig_fill(c, L, n, ctx_tables(c).C, SP, (const uint8_t *)META.p.get(), mode, d_item_mode, stream));
    c->share_passes++;
  }
  if (defer) HS_CUDA(c, cudaEventRecord(c->ev_tail[set], c->stream_tail));
  // a pass on a caller's stream: the next host-pointer call waits for it before it reuses this scratch (and group_digests, whose
  // Digest kernel hs_verify_groups_dev enqueued before this pass on the same stream)
  if (fin_stream != c->stream) HS_CUDA(c, cudaEventRecord(c->ev_dev_pass, fin_stream));
  return HS_OK;
}

// ---- the ring kernels' launches: each is the only launch of its kernel, counts it and returns the launch error
// k_verify_bulk (one thread per record) or k_verify_small (one block per record) over ring positions [base, base + n), completing
// with seq; the signature-cache instantiation when sc has a table.
template <bool SIGC>
static cudaError_t launch_ring_verify_as(hs_ctx *c, const ring_bufs &r, uint32_t mask, uint32_t base, uint32_t n, bool bulk,
                                         const committee_tables &C, const comb_params &cp, const sig_cache_dev &sc, uint32_t seq, cudaStream_t s) {
  if (bulk)
    k_verify_bulk<SIGC><<<blocks_for(n, HS_BULK_THREADS), HS_BULK_THREADS, 0, s>>>(r.recs.d, base, mask, n, c->d_btable, C, cp, r.flags.d, r.counters,
                                                                                 r.done.d, seq, sc);
  else
    k_verify_small<SIGC><<<n, 64, 0, s>>>(r.recs.d, base, mask, c->d_btable, C, cp, r.flags.d, r.counters, r.done.d, seq, sc);
  c->launches++;
  return cudaGetLastError();
}
static cudaError_t launch_ring_verify(hs_ctx *c, const ring_bufs &r, uint32_t mask, uint32_t base, uint32_t n, bool bulk, const committee_tables &C,
                                      const comb_params &cp, const sig_cache_dev &sc, uint32_t seq, cudaStream_t s) {
  return sc.b ? launch_ring_verify_as<true>(c, r, mask, base, n, bulk, C, cp, sc, seq, s)
              : launch_ring_verify_as<false>(c, r, mask, base, n, bulk, C, cp, sc, seq, s);
}
// k_queue_generic over the n ring slots listed in slots[] from position base on, the records' keys in pks.
static cudaError_t launch_queue_generic(hs_ctx *c, const ring_bufs &r, const uint8_t *pks, const uint32_t *slots, uint32_t mask, uint32_t base,
                                        uint32_t n, const comb_params &cp, uint32_t seq, cudaStream_t s) {
  k_queue_generic<<<blocks_for(n, HS_GEN_THREADS), HS_GEN_THREADS, 0, s>>>(r.recs.d, pks, slots, base, mask, n, c->d_btable, cp, r.flags.d,
                                                                         r.counters, r.done.d, seq);
  c->launches++;
  return cudaGetLastError();
}
// k_queue_digests over the n_desc descriptors in list from position base on: the Digests of their preimages into the records' msg.
static cudaError_t launch_queue_digests(hs_ctx *c, const ring_bufs &r, const qmsg_desc *list, uint32_t mask, uint32_t base, uint32_t n_desc,
                                        const uint8_t *arena, uint8_t *stage, uint32_t *digs, cudaStream_t s) {
  k_queue_digests<<<n_desc, HS_QDIG_THREADS, 0, s>>>(list, base, mask, arena, stage, digs, r.recs.d);
  c->launches++;
  return cudaGetLastError();
}
// The explain lane's share of the device: at most one block of HS_THREADS per HS_QUEUE_EXPLAIN_SM_DIV multiprocessors (33 blocks, 4,224
// records in flight, on a 132-SM H100).  A k_queue_explain block holds its SM's registers for a whole re-check (about 1.4 ms), so a
// large explain launch takes at most that share of the SMs from the verify launches; more records run grid-stride, one wave after another.
#define HS_QUEUE_EXPLAIN_SM_DIV 4
// k_queue_explain over the n records of the n_desc requests in list, reading their regions from mirror, writing why bytes and
// completion words into the mapped arena.
static cudaError_t launch_queue_explain(hs_ctx *c, const xq_desc *list, uint32_t n_desc, uint32_t n, uint8_t *mirror, uint8_t *arena,
                                        cudaStream_t s) {
  const unsigned grid = (unsigned)std::min<size_t>(blocks_for(n), std::max<size_t>(1, c->n_sms / HS_QUEUE_EXPLAIN_SM_DIV));
  k_queue_explain<<<grid, HS_THREADS, 0, s>>>(list, n_desc, n, mirror, arena);
  c->launches++;
  return cudaGetLastError();
}
// k_sig_audit over buckets [first, first + n) of table b, results into out (4 words).  Its threads run explain_record's re-check as the
// explain lane's do, so it takes the same share of the SMs.
static cudaError_t launch_sig_audit(hs_ctx *c, sig_bucket *b, uint32_t first, uint32_t n, unsigned long long *out, cudaStream_t s) {
  const unsigned grid = (unsigned)std::min<size_t>(blocks_for((size_t)n * HS_SIG_WAYS), std::max<size_t>(1, c->n_sms / HS_QUEUE_EXPLAIN_SM_DIV));
  k_sig_audit<<<grid, HS_THREADS, 0, s>>>(b, first, n, out);
  c->launches++;
  return cudaGetLastError();
}

// ---- latency path (host side)
// key bytes -> table index through the host mirror of the device hash table (registered committee or learned cache)
static uint32_t host_key_lookup(const hs_ctx *c, const uint8_t *key) {
  return c->h_index.find(c->h_pks.data(), key, [c](uint32_t idx) { return idx < c->n_keys; });
}
static bool small_eligible(const hs_ctx *c, size_t n) { return c->small_enabled && n >= 1 && n <= HS_SMALL_MAX && has_key_tables(c); }
// Record i of a latency-path call: its signature, its 32-byte message and its key's table index.
struct small_src {
  const uint8_t *sig, *msg;
  uint32_t vidx;
};
// Fills c->small.recs.h[0 .. n) from rec(i) and reports whether every key index resolved (!= HS_NO_KEY).
template <class Rec>
static bool small_stage(hs_ctx *c, size_t n, Rec rec) {
  bool all = true;
  for (size_t i = 0; i < n; i++) {
    const small_src s = rec(i);
    memcpy(c->small.recs.h[i].sig, s.sig, 64);
    memcpy(c->small.recs.h[i].msg, s.msg, 32);
    c->small.recs.h[i].vidx = s.vidx;
    all = all && s.vidx != HS_NO_KEY;
  }
  return all;
}
// c->small.recs.h[0 .. n) is filled: one launch (one request in slot 0), then poll the completion word the last block writes to
// mapped host memory.
static int run_small(hs_ctx *c, size_t n, uint32_t mode, uint32_t *out_bitmap) {
  for (size_t i = 0; i < n; i++) {
    c->small.recs.h[i].req = 0;
    c->small.recs.h[i].req_n = (uint32_t)n;
  }
  const uint32_t seq = ++c->small_seq ? c->small_seq : ++c->small_seq;  // never 0
  HS_TRY(wait_key_cache_build(c, c->stream));
  HS_CUDA(c, launch_ring_verify(c, c->small, HS_SMALL_MAX - 1, 0, (uint32_t)n, false, ctx_tables(c).C, c->cp, sig_cache_dev{}, seq, c->stream));
  volatile uint32_t *done = c->small.done.h;
  bool finished = false;
  for (uint64_t spin = 0; spin < (1ull << 34); spin++) {
    if (*done == seq) {
      finished = true;
      break;
    }
    if ((spin & 0xfff) == 0xfff) {
      cudaError_t q = cudaStreamQuery(c->stream);
      if (q != cudaSuccess && q != cudaErrorNotReady) return fail(c, HS_ERR_CUDA, "k_verify_small", q);
      if (q == cudaSuccess && *done != seq && spin > (1u << 20)) break;  // stream drained without the completion word
    }
  }
  if (!finished) {
    HS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (*done != seq) return fail(c, HS_ERR_CUDA, "k_verify_small did not complete");
  }
  for (size_t w = 0; w < (n + 31) / 32; w++) out_bitmap[w] = 0;
  const uint32_t want = mode_flag(mode);
  for (size_t i = 0; i < n; i++)
    if (((volatile uint8_t *)c->small.flags.h)[i] & want) out_bitmap[i >> 5] |= 1u << (i & 31);
  return HS_OK;
}

// ---- verify queue (hs_queue_*): continuous batching of concurrent small verifies onto k_verify_small
// Ring positions grow without bound (slot = position & mask): [head, launched) is dispatched, [launched, tail) pending.  A
// request's slot is the ring slot of its first record; it names the request's counter, completion word and bookkeeping.
// The dispatcher thread is the only one that launches, watches completions, runs the slow path and advances `head`.
// A request is either small (hs_queue_submit: 1..64 records, one mode) or a group (hs_queue_submit_group: one consensus
// message's certificate, up to the ring's capacity, a mode per record); both take the same ring, launches and completion path.
#define HS_QUEUE_DEFAULT_RECORDS 4096u
#define HS_QUEUE_MAX_RECORDS (1u << 20)
#define HS_QUEUE_MAX_INFLIGHT 2  // k_verify_small launches; bulk launches do not count against it
// Device requests of at least this many records get their own k_verify_bulk launch on the queue's second stream: the smallest
// measured Block certificate from which one thread per signature plus a block-level inversion was no slower than k_verify_small's
// block per signature (1,002 records, N = 1,500: 345 vs 375 us p50; at 668 records 307 vs 298 us; DESIGN.md §5d).
#define HS_QUEUE_BULK_MIN 1002
static_assert(HS_QUEUE_BULK_MIN > HS_SMALL_MAX, "small requests never take the bulk path");
// Preimage arena bytes per ring record: a full ring of 16-byte TC preimages with their offsets and indices (28 bytes a record), or
// a Block preimage with about a thousand payload digests.
#define HS_QUEUE_ARENA_PER_RECORD 64u
// A request's verdict bitmap: inline for <= 64 records (every small request), on the heap only for larger groups.
struct queue_bits {
  uint32_t inl[(HS_SMALL_MAX + 31) / 32] = {0, 0};
  std::vector<uint32_t> big;
  void set(uint32_t n, const uint32_t *src_or_null) {  // null: all zero (a failed request rejects every record)
    const size_t w = (n + 31) / 32;
    uint32_t *d = inl;
    if (n > HS_SMALL_MAX) {
      big.assign(w, 0);
      d = big.data();
    } else {
      inl[0] = inl[1] = 0;
    }
    if (src_or_null) memcpy(d, src_or_null, 4 * w);
  }
  const uint32_t *data() const { return big.empty() ? inl : big.data(); }
};
// Where a request's verdicts go: its callback, or the results entry of its ticket when cb is null.  Every request kind opens and
// closes its ticket through ticket_open_locked / ticket_close_locked.
struct ticket_sink {
  size_t ticket;
  hs_queue_cb *cb;
  void *user;
};
// A byte arena of cap bytes (a power of two) whose positions grow without bound like the ring's: [head, tail) is in use, and a
// position's offset is position & (cap - 1).  A region is contiguous: one that would cross the arena's end starts at its beginning.
struct byte_ring {
  uint64_t cap = 0, head = 0, tail = 0;
  // The start position of a free region of `size` <= cap bytes, or none when the arena has no room now.  Commits nothing (an empty
  // arena may only move its start): the caller sets tail past the region once its request is accepted.
  std::optional<uint64_t> take(uint64_t size) {
    uint64_t start = tail;
    if (off(start) + size > cap) start += cap - off(start);  // would cross the end: start over
    if (start + size - head > cap) {                       // arena full
      if (head != tail) return std::nullopt;
      head = tail = start;  // empty: the skipped tail is free too
    }
    return start;
  }
  void release_to(uint64_t end) { head = std::max(head, end); }
  uint64_t off(uint64_t pos) const { return pos & (cap - 1); }
};
// Certificate cache (hs_queue_cert_cache).  A span is the batch-eq records of one request that sign the same message, at least two
// of them: a QC's votes.  Its key is a kind byte ('P': a preimage of hs_queue_submit_msgs, 'D': a Digest of hs_queue_submit_group),
// the message's length and bytes, then (pk | sig) of each record in request order; lookups go through a hash of the key and match
// only on equal bytes.  A span that verified in full is kept (least recently used first out, up to max_bytes of keys) and answers 1
// for every record of an identical span later.  An identical span still pending or in flight is joined: the later request puts
// none of those records in the ring and takes the earlier request's bits and status for them.
struct cert_key {
  size_t h;
  std::string_view k;
  bool operator==(const cert_key &o) const { return h == o.h && k == o.k; }
};
struct cert_key_hash {
  size_t operator()(const cert_key &x) const { return x.h; }
};
struct cert_span {
  std::string key;
  size_t h;
  std::vector<uint32_t> idx;  // its records in the request, in request order
  uint8_t role;               // CERT_NEW (its records enter the ring: this request is its primary), CERT_HIT or CERT_JOINED
};
enum { CERT_NEW, CERT_HIT, CERT_JOINED };
// A request submitted with the cache on that has at least one span.  It completes when its ring part (the records that entered
// the ring, if any) and every span it joined are done: `pending` counts them.
struct cert_req {
  ticket_sink sink;
  uint32_t n;
  std::vector<cert_span> spans;
  std::vector<uint32_t> ring_idx;  // the request's record of each ring record of its ring part
  uint32_t pending = 0;
  int status = HS_OK;
  std::vector<uint32_t> bits;  // n verdict bits
};
struct cert_flight {  // the identical spans waiting on a span its primary request is verifying
  std::vector<std::pair<cert_req *, const cert_span *>> joiners;
};
// hs_queue_generic's lists (allocated whole on first use): a generic launch's ring slots at positions [lo, lo + records), and its
// preimage requests' descriptors from position lo on.
struct generic_lists {
  mapped<uint32_t> slot;
  mapped<qmsg_desc> mlist;
};
// hs_queue_sig_cache's bucket-mix key and HS_SIG_CTRS counters per ring slot, on the device and mapped (allocated whole on first use).
struct sig_counters {
  dev_mem<uint64_t> key;
  dev_mem<uint32_t> ctr;
  mapped<uint32_t> hctr;
};
// ---- side lanes of the verify queue: the batch lane (hs_queue_batch) and the explain lane (hs_queue_explain)
// A side lane's requests never enter the ring.  Each takes a region of the lane's mapped arena under q->mu and is filled outside it:
// inputs, then result words, then a 16-byte tail whose word [1] is the completion word.  One launch is in flight per lane, on the lane's
// own streams; it takes the ready requests at the front of the lane's list, and each request completes when its completion word
// carries the launch's number.  The functions below serve both lanes; what differs is the lane_kind.
struct side_lane;
struct lane_kind {
  const char *name;                          // in the lane's error texts
  const char *configure;                     // the entry point that turns it on
  size_t per_launch;                         // requests one launch takes at most
  const char *launch_err, *incomplete;       // texts of a failed stream and of a completion word missing on drained streams
  int (*enqueue)(hs_queue *q, side_lane &L);  // enqueues the launch of L.launch on the lane's streams (under c->mu)
  void (*count)(hs_queue *q, side_lane &L);  // counts a launch whose every request completed HS_OK (under q->mu)
};
static int batch_enqueue(hs_queue *q, side_lane &L);
static void batch_count(hs_queue *q, side_lane &L);
static int explain_enqueue(hs_queue *q, side_lane &L);
static void explain_count(hs_queue *q, side_lane &L);
static const lane_kind batch_kind{"batch", "hs_queue_batch", 1, "verify queue batch pass", "verify queue: k_batch_done did not complete",
                                  batch_enqueue, batch_count};
static const lane_kind explain_kind{"explain", "hs_queue_explain", SIZE_MAX, "verify queue explain launch",
                                    "verify queue: k_queue_explain did not complete", explain_enqueue, explain_count};
struct lane_req {
  ticket_sink sink;
  uint32_t n_bits;                // the ticket's verdict bits
  uint32_t n, m, n_groups;        // the launch's shape: records (items), messages (preimages), groups,
  uint64_t pre_bytes;             //   preimage bytes
  uint64_t o_res, o_tail, size;   // its result words, its tail and its size, from the lane's region layout
  uint64_t a_off = 0, a_pos = 0, a_end = 0;  // region offset in the arena; arena positions of its start and past its end
  uint32_t seq = 0;               // the completion word (set at launch)
  uint32_t share_gen = 0;         // batch lane: the signature-cache table its pass shared (0: none; set at launch)
  bool ready = false, done = false;
};
// A side lane's arena, its device mirror and its streams (lane_configure builds them whole, or not at all).
struct lane_bufs {
  mapped<uint8_t> arena;    // request regions
  dev_mem<uint8_t> mirror;  // the inputs of the regions in flight, at the same offsets
  stream_h stream, side;    // the lane's stream (the device's lowest priority) and, for the batch lane, its miss pass's stream
};
// Off while max_recs is 0.  Requests wait in reqs in submit order.  launch is the requests of the launch in flight (dispatcher thread;
// changed under q->mu).  The buffers change only while the lane is off and reqs is empty.
struct side_lane {
  explicit side_lane(const lane_kind &k) : kind(k) {}
  const lane_kind &kind;
  size_t max_recs = 0, max_bytes = 0;  // limits of one request
  byte_ring ring;                      // positions in buf.arena
  lane_bufs buf;
  std::deque<lane_req> reqs;
  std::vector<lane_req *> launch;
  uint32_t seq = 0;
  uint64_t stats[HS_QUEUE_BATCH_STATS] = {};  // hs_queue_batch_stats / hs_queue_explain_stats
  std::mutex cfg_mu;                          // serialises the lane's configure calls
};
static_assert(HS_QUEUE_EXPLAIN_STATS <= HS_QUEUE_BATCH_STATS, "a lane's stats array holds either lane's counters");
// The batch lane's own scratch: the pass's Digests, hs_verify_groups' per-item buffers and the miss pass's events.
struct batch_scratch {
  dev_mem<uint32_t> dig;  // the request's Digests, 32 bytes per preimage
  dev_mem<fe> xyz;
  dev_mem<uint8_t> meta;
  dev_mem<uint32_t> vidx, miss, miss_count, items, grej, counter;
  event_h ev[2];
  // a pass that shares the queue's signature cache (hs_queue_sig_share): its miss list, flag bytes, device counters (HS_SIG_CTRS, then
  // the list's count) and the mapped copy of the counts
  dev_mem<uint32_t> share_list, share_ctr;
  dev_mem<uint8_t> share_fl;
  mapped<uint32_t> share_h;
};
// The explain lane's own scratch: the launch's request list.
struct explain_scratch {
  mapped<xq_desc> list;
};
struct hs_queue {
  hs_ctx *c = nullptr;
  uint32_t cap = 0, mask = 0;
  ring_bufs ring;                        // cap slots
  mapped<uint8_t> pk;                   // key bytes per record (32 B; resolved to a table index at dispatch, read by k_queue_generic)
  std::vector<uint8_t> modes;            // HS_MODE_* per record (host only: picks the verdict flag of each record)
  std::vector<uint32_t> wbits;           // dispatcher thread only: verdict bitmap being assembled (cap bits)
  stream_h stream;                       // k_verify_small launches: the device's highest priority
  stream_h bulk_stream;                  // k_verify_bulk launches: a lower priority, so votes never wait behind them
  event_h ev_last;                       // recorded after every launch on `stream`: the ring is freed only after it
  event_h ev_bulk_last;                  // the same for `bulk_stream`
  uint64_t stats[HS_QUEUE_STATS] = {};   // hs_queue_stats
  // preimage requests (hs_queue_submit_msgs): a byte arena of HS_QUEUE_ARENA_PER_RECORD x cap bytes; a request's region is
  // released with its ring slots
  byte_ring arena;
  mapped<uint8_t> arena_buf;             // the requests' regions (layout: qmsg_desc)
  dev_mem<uint8_t> d_stage;              // k_queue_digests' copy of the arena (same offsets)
  dev_mem<uint32_t> d_digs;              // digest slots, 32 bytes per 8 arena bytes
  mapped<qmsg_desc> mlist;               // a launch's descriptors at the ring slots of its range
  uint64_t dstats[HS_QUEUE_DIGEST_STATS] = {};     // hs_queue_digest_stats
  struct req {
    ticket_sink sink;
    uint32_t n;
    uint32_t seq;   // launch that verifies it (0: slow path)
    bool finished;
    bool msgs;           // a preimage request: its records' Digests are computed by k_queue_digests
    uint32_t a_off, m, pre_bytes;  // its arena region: offset, preimages, preimage bytes
    uint64_t a_end;      // arena position past its region (0: none)
    cert_req *cr = nullptr;  // the ring part of a certificate-cache request: its verdicts go there (sink unused)
    bool gen = false;        // set at dispatch: verified by k_queue_generic (hs_queue_generic on, a key outside the committee)
  };
  std::vector<req> reqs;  // by request slot
  struct result {
    bool done;
    int status;
    uint32_t n;
    queue_bits bits;
  };
  std::unordered_map<size_t, result> results;  // tickets without a callback, until poll / wait reads them
  struct launch {
    uint32_t seq;
    uint64_t lo, hi;  // ring positions it covers
    bool bulk;        // on bulk_stream: k_verify_bulk (one request) or k_queue_generic; else k_verify_small on stream
    uint32_t sig_gen;  // the signature cache's table it probed (0: launched without the cache)
    bool generic = false;  // k_queue_generic: its requests are the gen ones in [lo, hi) with its seq, others lie between them
  };
  // Launches in flight, in launch order.  A generic launch's range interleaves with small and bulk ones, so this is not ring
  // order: queue_release_locked takes the lowest lo of all of them.
  std::deque<launch> inflight;
  // hs_queue_generic: gen_on is written under c->mu (the dispatcher reads it there); at most one generic launch is in flight, and
  // generic requests dispatched meanwhile wait in gpend (ring positions, dispatcher thread only) for the next one
  std::atomic<bool> gen_on{false};
  std::deque<uint64_t> gpend;
  generic_lists gen_bufs;
  uint64_t gstats[HS_QUEUE_GENERIC_STATS] = {};      // hs_queue_generic_stats
  side_lane batch{batch_kind}, explain{explain_kind};  // the side lanes (dispatched in this order, ahead of ring work)
  batch_scratch batch_scr;
  explain_scratch explain_scr;
  uint64_t head = 0, launched = 0, tail = 0;
  size_t next_ticket = 1;
  uint32_t seq = 0;
  uint64_t spins = 0;
  bool stop = false;
  // certificate cache (hs_queue_cert_cache): off while cc_max is 0
  std::atomic<size_t> cc_max{0};
  size_t cc_bytes = 0;                                // key bytes held
  std::list<std::pair<std::string, size_t>> cc_lru;  // verified span keys and their hashes, most recently used first
  std::unordered_map<cert_key, std::list<std::pair<std::string, size_t>>::iterator, cert_key_hash> cc_map;
  std::unordered_map<cert_key, cert_flight, cert_key_hash> cc_flights;  // keyed by the primary's span key
  std::vector<cert_req *> cc_ready;  // answered entirely at submit: the queue's thread completes them
  uint64_t cstats[HS_QUEUE_CERT_STATS] = {};  // hs_queue_cert_stats ([5] is cc_bytes)
  // signature cache (hs_queue_sig_cache): off while d_sig is null.  The table, its key and bmask change only under c->mu after
  // both streams drained; sig_gen (also under mu) numbers the tables, so counts of a replaced table's launches are not held.
  dev_mem<sig_bucket> d_sig;
  uint32_t sig_bmask = 0, sig_gen = 0;
  sig_counters sigc;
  uint64_t sstats[HS_QUEUE_SIG_STATS] = {};  // hs_queue_sig_stats ([4]: inserts - evictions into the current table)
  // hs_queue_sig_share: ev_share is recorded after every batch-lane pass that shares the table (under c->mu), so a resize can wait for it
  event_h ev_share;
  uint64_t shstats[HS_QUEUE_SIG_SHARE_STATS] = {};  // hs_queue_sig_share_stats
  // hs_queue_sig_audit: ev_audit is recorded after every audit launch on the table (under c->mu), so a resize can wait for it; d_audit
  // holds a launch's four result words (audits run one at a time under c->audit_mu)
  event_h ev_audit;
  dev_mem<unsigned long long> d_audit;
  uint64_t astats[HS_QUEUE_SIG_AUDIT_STATS] = {};  // hs_queue_sig_audit_stats
  std::mutex mu;  // everything above that submit / poll / wait touch: tail, reqs of pending slots, results, head, stop
  std::condition_variable cv_work, cv_done;
  std::thread th;
};

// ---- hs_queue_sig_share: the host-pointer verify calls and the batch lane share one queue's signature cache
// The counts of one shared pass (h: its mapped HS_SIG_CTRS words, complete) into q's counters, under q->mu; gen: the table it shared.
static void sig_share_count(hs_queue *q, const uint32_t *h, uint32_t gen) {
  const volatile uint32_t *v = h;
  for (int k = 0; k < HS_SIG_CTRS; k++) q->shstats[k] += v[k];
  q->shstats[4]++;
  if (gen == q->sig_gen) q->sstats[4] += v[2] - v[3];
}
// Set on every verify queue's dispatcher thread: the synchronous calls it makes for slow-path requests neither probe nor insert.
static thread_local bool t_queue_dispatcher = false;
// Held, under c->mu, by each host-pointer call that takes part (hs_verify_rec128, hs_verify_batch_shared_msg, hs_verify_qcs,
// hs_verify_tcs, hs_verify_groups): while it lives, run_verify's committee pass over 32-byte messages on the context's stream shares the
// table of c->share_q.  Each of these calls runs at most one such pass; once its results are back its counts go to the queue.
struct share_call {
  hs_ctx *c;
  explicit share_call(hs_ctx *ctx) : c(ctx) {
    hs_queue *q = c->share_q;
    c->share_passes = 0;
    c->share_sc = (q && !t_queue_dispatcher) ? sig_cache_dev{q->d_sig, q->sigc.key, q->sig_bmask, c->share_ctr, nullptr} : sig_cache_dev{};
  }
  ~share_call() {
    if (c->share_passes && cudaStreamSynchronize(c->stream) == cudaSuccess) {
      std::lock_guard<std::mutex> g(c->share_q->mu);
      sig_share_count(c->share_q, c->share_h.h, c->share_q->sig_gen);
    }
    c->share_sc = sig_cache_dev{};
  }
};

struct queue_completion {
  hs_queue_cb *cb;
  void *user;
  size_t ticket;
  int status;
  queue_bits bits;
};
// Issues ticket s.ticket, which is q->next_ticket, to a request just accepted (under q->mu): a polled ticket parks its results
// entry of n_bits verdict bits.  A callback ticket never touches `results`.
static void ticket_open_locked(hs_queue *q, const ticket_sink &s, uint32_t n_bits) {
  q->next_ticket++;
  if (!s.cb) q->results[s.ticket] = hs_queue::result{false, HS_OK, n_bits, {}};
}
// Completes ticket s (under q->mu) with n_bits verdict bits, all zero unless status is HS_OK (a failed request rejects every
// record): its callback is returned in `fire`, to run after the lock is released, or its parked result is filled.
static void ticket_close_locked(hs_queue *q, const ticket_sink &s, int status, uint32_t n_bits, const uint32_t *bits,
                                std::vector<queue_completion> &fire) {
  if (status != HS_OK) bits = nullptr;
  if (s.cb) {
    fire.push_back(queue_completion{s.cb, s.user, s.ticket, status, {}});
    fire.back().bits.set(n_bits, bits);
  } else {
    hs_queue::result &res = q->results[s.ticket];
    res.done = true;
    res.status = status;
    res.bits.set(n_bits, bits);
    q->cv_done.notify_all();
  }
}
// Releases the ring space of the finished requests at the head — but never inside the range of a launch still in flight: its
// blocks may still read those records (slow-path requests between two device requests ride along in the launch).  The limit is
// the lowest range start of ALL launches in flight: a generic launch's range holds requests of other launches, and its slot list
// sits at its own positions, so finished requests inside it must not be released either.  Generic requests waiting in gpend are
// unfinished, so release stops at them without a limit.
static void queue_release_locked(hs_queue *q) {
  uint64_t limit = q->launched;
  for (const hs_queue::launch &L : q->inflight) limit = std::min(limit, L.lo);
  while (q->head < limit && q->reqs[q->head & q->mask].finished) {
    hs_queue::req &h = q->reqs[q->head & q->mask];
    h.finished = false;
    q->head += h.n;
    q->arena.release_to(h.a_end);
  }
}
// Completes a certificate-cache request whose parts are all done (under q->mu).
static void cert_complete_locked(hs_queue *q, cert_req *cr, std::vector<queue_completion> &fire) {
  ticket_close_locked(q, cr->sink, cr->status, cr->n, cr->bits.data(), fire);
  delete cr;
}
static void cert_evict_locked(hs_queue *q, size_t limit) {  // least recently used first out, until at most `limit` bytes are held
  while (q->cc_bytes > limit) {
    const auto &b = q->cc_lru.back();
    q->cc_map.erase(cert_key{b.second, b.first});
    q->cc_bytes -= b.first.size();
    q->cc_lru.pop_back();
  }
}
static void cert_insert_locked(hs_queue *q, std::string &&key, size_t h) {
  const size_t max = q->cc_max.load();
  if (key.size() > max || q->cc_map.count(cert_key{h, key})) return;
  cert_evict_locked(q, max - key.size());
  q->cc_bytes += key.size();
  q->cc_lru.emplace_front(std::move(key), h);
  q->cc_map.emplace(cert_key{h, q->cc_lru.front().first}, q->cc_lru.begin());
  q->cstats[4]++;
}
// The ring part of certificate-cache request cr is done (bits: its ring records' verdicts, null on error).  Each span it verified
// hands its bits and status to the requests that joined it, and enters the cache if every one of its records verified.
static void cert_part_done_locked(hs_queue *q, cert_req *cr, int status, const uint32_t *bits, std::vector<queue_completion> &fire) {
  if (status != HS_OK) cr->status = status;
  else
    for (size_t k = 0; k < cr->ring_idx.size(); k++)
      if ((bits[k >> 5] >> (k & 31)) & 1u) cr->bits[cr->ring_idx[k] >> 5] |= 1u << (cr->ring_idx[k] & 31);
  for (cert_span &sp : cr->spans) {
    if (sp.role != CERT_NEW) continue;
    bool all = status == HS_OK;
    for (uint32_t i : sp.idx) all = all && ((cr->bits[i >> 5] >> (i & 31)) & 1u);
    auto it = q->cc_flights.find(cert_key{sp.h, sp.key});
    for (auto &[jr, js] : it->second.joiners) {
      if (status != HS_OK) jr->status = status;
      else
        for (size_t t = 0; t < sp.idx.size(); t++)
          if ((cr->bits[sp.idx[t] >> 5] >> (sp.idx[t] & 31)) & 1u) jr->bits[js->idx[t] >> 5] |= 1u << (js->idx[t] & 31);
      if (--jr->pending == 0) cert_complete_locked(q, jr, fire);
    }
    q->cc_flights.erase(it);
    if (all) cert_insert_locked(q, std::move(sp.key), sp.h);
  }
  if (--cr->pending == 0) cert_complete_locked(q, cr, fire);
}

// Marks the request at ring position p finished (under q->mu) and completes its ticket, or its certificate-cache request's ring part.
static void queue_finish_locked(hs_queue *q, uint64_t p, int status, const uint32_t *bits, std::vector<queue_completion> &fire) {
  hs_queue::req &r = q->reqs[p & q->mask];
  r.finished = true;
  if (r.cr) {
    cert_part_done_locked(q, r.cr, status, status == HS_OK ? bits : nullptr, fire);
    r.cr = nullptr;
  } else {
    ticket_close_locked(q, r.sink, status, r.n, bits, fire);
  }
  queue_release_locked(q);
}
static void queue_fire(std::vector<queue_completion> &fire) {
  for (queue_completion &f : fire) f.cb(f.user, f.ticket, f.status, f.bits.data());
  fire.clear();
}

// The Digests of one launch's preimage requests, on the launch's stream ahead of its verify: the descriptors of the preimage requests
// among those at positions ps go to `list` from position lo on, and one k_queue_digests launch takes them.  dig counts what was
// enqueued: launches, preimages and preimage bytes (hs_queue_digest_stats).
static cudaError_t queue_digests(hs_queue *q, mapped<qmsg_desc> &list, uint64_t lo, const std::vector<uint64_t> &ps, cudaStream_t s,
                                 uint64_t (&dig)[3]) {
  uint32_t n_desc = 0;
  uint64_t n_pre = 0, n_pre_bytes = 0;
  for (uint64_t p : ps) {
    const hs_queue::req &r = q->reqs[p & q->mask];
    if (!r.msgs) continue;
    list.h[(lo + n_desc++) & q->mask] = qmsg_desc{r.a_off, r.m, r.n, (uint32_t)(p & q->mask), r.pre_bytes, {0, 0, 0}};
    n_pre += r.m;
    n_pre_bytes += r.pre_bytes;
  }
  if (n_desc == 0) return cudaSuccess;
  const cudaError_t e =
      launch_queue_digests(q->c, q->ring, list.d, q->mask, (uint32_t)(lo & q->mask), n_desc, q->arena_buf.d, q->d_stage, q->d_digs, s);
  if (e == cudaSuccess) {
    dig[0]++;
    dig[1] += n_pre;
    dig[2] += n_pre_bytes;
  }
  return e;
}

// Dispatches the pending requests [lo, hi): under c->mu, keys are resolved through the host mirror of the key hash table and
// one launch covers every request whose keys are all registered; the others then run through hs_verify_rec128 on this thread.
// A slow-path request of at most 64 records between two device requests rides along in the launch (its blocks find no table
// index and reject; its verdicts are ignored).  A larger one would cost thousands of wasted blocks, so the launch is split
// around it: one launch per run of device requests between such requests.  A device request of HS_QUEUE_BULK_MIN records or more
// closes the run the same way and gets a k_verify_bulk launch of its own on the bulk stream; the small launches of the same
// dispatch are enqueued first.
// With hs_queue_generic on, a request with a key outside the committee (every request, when none is registered) is a generic
// request instead: it neither rides nor reaches the slow path.  It closes the run before it like a large rider, whatever its
// size (k_verify_small must not touch its records: they complete through k_queue_generic's counts), and waits in gpend.  When no
// generic launch is in flight, one k_queue_generic launch on the bulk stream, after this dispatch's other launches, takes every
// request in gpend.  Requests left in gpend after the option is turned off take the slow path.
static void queue_dispatch(hs_queue *q, uint64_t lo, uint64_t hi) {
  hs_ctx *c = q->c;
  std::vector<uint64_t> slow;
  std::vector<uint64_t> greqs;  // the requests of this dispatch's generic launch, in ring order
  hs_queue::launch G{0, 0, 0, true, 0, true};
  uint64_t g_recs = 0;
  bool g_ok = false;
  std::vector<queue_completion> fire;
  std::vector<hs_queue::launch> runs;  // ring ranges [lo, hi) to launch, first device request to past the last one, in ring order
  std::vector<char> ok;                // runs launched without a CUDA error (the first failure stops the rest)
  std::vector<uint64_t> dev;           // the device-path requests of the run being launched (slow-path riders carry no digest)
  uint64_t dig_launched[3] = {0, 0, 0};  // k_queue_digests launches, their preimages and preimage bytes (hs_queue_digest_stats)
  cudaError_t e = cudaSuccess;
  {
    std::lock_guard<std::mutex> g(c->mu);
    const bool committee = committee_registered(c) && c->small_enabled;
    const bool gen = q->gen_on.load();  // hs_queue_generic writes it under c->mu
    if (!gen) {  // turned off with generic requests still waiting: they take the slow path, ahead of this range's
      for (uint64_t p : q->gpend) q->reqs[p & q->mask].gen = false;
      slow.assign(q->gpend.begin(), q->gpend.end());
      q->gpend.clear();
    }
    uint64_t rlo = hi, rhi = lo;  // the run being gathered
    for (uint64_t p = lo; p < hi;) {
      hs_queue::req &r = q->reqs[p & q->mask];
      bool all = committee;
      for (uint32_t i = 0; i < r.n; i++) {
        small_rec &s = q->ring.recs.h[(p + i) & q->mask];
        s.vidx = all ? host_key_lookup(c, q->pk.h + 32 * (size_t)((p + i) & q->mask)) : HS_NO_KEY;
        s.req = (uint32_t)(p & q->mask);
        s.req_n = r.n;
        if (s.vidx == HS_NO_KEY) all = false;
      }
      const bool bulk = all && r.n >= HS_QUEUE_BULK_MIN;
      const bool generic = gen && !all;
      r.gen = generic;
      if (!all) {  // every record of a slow-path request rides as HS_NO_KEY: none of them probes or fills the signature cache
        for (uint32_t i = 0; i < r.n; i++) q->ring.recs.h[(p + i) & q->mask].vidx = HS_NO_KEY;
        r.seq = 0;  // a generic request's launch number is set when its launch is built
        if (generic) q->gpend.push_back(p);
        else slow.push_back(p);
      } else {
        r.seq = 1;  // the launch's number is set below
      }
      // no large riders, no generic request in a small launch, and no small request in a bulk launch
      if ((bulk || (!all && (generic || r.n > HS_SMALL_MAX))) && rlo < rhi) {
        runs.push_back(hs_queue::launch{0, rlo, rhi, false});
        rlo = hi;
        rhi = lo;
      }
      if (bulk) {
        runs.push_back(hs_queue::launch{0, p, p + r.n, true});
      } else if (all) {
        if (rlo == hi) rlo = p;
        rhi = p + r.n;
      }
      p += r.n;
    }
    if (rlo < rhi) runs.push_back(hs_queue::launch{0, rlo, rhi, false});
    const committee_tables C = ctx_tables(c).C;
    const sig_cache_dev sc = q->d_sig ? sig_cache_dev{q->d_sig, q->sigc.key, q->sig_bmask, q->sigc.ctr, q->sigc.hctr.d} : sig_cache_dev{};
    ok.assign(runs.size(), 0);
    for (int pass = 0; pass < 2 && e == cudaSuccess; pass++) {  // pass 0: the small launches, pass 1: the bulk ones
      for (size_t k = 0; k < runs.size(); k++) {
        hs_queue::launch &L = runs[k];
        if (L.bulk != (pass == 1)) continue;
        L.seq = ++q->seq ? q->seq : ++q->seq;  // never 0
        L.sig_gen = q->d_sig ? q->sig_gen : 0;
        dev.clear();
        for (uint64_t p = L.lo; p < L.hi; p += q->reqs[p & q->mask].n) {
          hs_queue::req &r = q->reqs[p & q->mask];
          if (!r.seq) continue;
          r.seq = L.seq;
          dev.push_back(p);
        }
        cudaStream_t s = L.bulk ? q->bulk_stream : q->stream;
        e = queue_digests(q, q->mlist, L.lo, dev, s, dig_launched);
        if (e == cudaSuccess)
          e = launch_ring_verify(c, q->ring, q->mask, (uint32_t)(L.lo & q->mask), (uint32_t)(L.hi - L.lo), L.bulk, C, c->cp, sc, L.seq, s);
        if (e == cudaSuccess) e = L.bulk ? cudaEventRecord(q->ev_bulk_last, q->bulk_stream) : cudaEventRecord(q->ev_last, q->stream);
        if (e != cudaSuccess) {
          fail(c, HS_ERR_CUDA, "verify queue launch", e);
          break;
        }
        ok[k] = 1;
      }
    }
    bool g_inflight = false;  // (inflight changes only on this thread)
    for (const hs_queue::launch &L : q->inflight) g_inflight = g_inflight || L.generic;
    if (gen && !g_inflight && !q->gpend.empty()) {  // the generic launch: its slot list and descriptors start at position lo
      greqs.assign(q->gpend.begin(), q->gpend.end());
      q->gpend.clear();
      G.seq = ++q->seq ? q->seq : ++q->seq;
      G.lo = greqs.front();
      for (uint64_t p : greqs) {
        hs_queue::req &r = q->reqs[p & q->mask];
        r.seq = G.seq;
        for (uint32_t i = 0; i < r.n; i++) q->gen_bufs.slot.h[(G.lo + g_recs++) & q->mask] = (uint32_t)((p + i) & q->mask);
        G.hi = p + r.n;
      }
      const bool earlier_failure = e != cudaSuccess;
      if (e == cudaSuccess) e = queue_digests(q, q->gen_bufs.mlist, G.lo, greqs, q->bulk_stream, dig_launched);
      if (e == cudaSuccess)
        e = launch_queue_generic(c, q->ring, q->pk.d, q->gen_bufs.slot.d, q->mask, (uint32_t)(G.lo & q->mask), (uint32_t)g_recs, c->cp, G.seq,
                                 q->bulk_stream);
      if (e == cudaSuccess) e = cudaEventRecord(q->ev_bulk_last, q->bulk_stream);
      g_ok = e == cudaSuccess;
      if (!g_ok && !earlier_failure) fail(c, HS_ERR_CUDA, "verify queue generic launch", e);
    }
  }
  {
    std::lock_guard<std::mutex> g(q->mu);
    if (!greqs.empty()) {
      if (g_ok) {
        q->inflight.push_back(G);
        q->gstats[0]++;
        q->gstats[1] += g_recs;
        q->gstats[2] += greqs.size();
      } else {
        for (uint64_t p : greqs) queue_finish_locked(q, p, HS_ERR_CUDA, nullptr, fire);
      }
    }
    for (uint64_t p : slow) {
      q->stats[4]++;
      q->stats[5] += q->reqs[p & q->mask].n;
    }
    for (int i = 0; i < 3; i++) q->dstats[i] += dig_launched[i];
    for (size_t k = 0; k < runs.size(); k++) {
      const hs_queue::launch &L = runs[k];
      if (ok[k]) {
        q->inflight.push_back(L);
        q->stats[L.bulk ? 2 : 0]++;
        q->stats[L.bulk ? 3 : 1] += L.hi - L.lo;
      } else {
        for (uint64_t p = L.lo; p < L.hi; p += q->reqs[p & q->mask].n)
          if (q->reqs[p & q->mask].seq) queue_finish_locked(q, p, HS_ERR_CUDA, nullptr, fire);
      }
    }
  }
  queue_fire(fire);
  // the slow path: exactly the synchronous entry point (key cache, generic kernels), on this thread — one call per verdict mode
  // present in the request (a small request has one mode; a Block group has a strict pass and a batch-eq pass)
  std::vector<hs_rec128> recs;
  std::vector<uint32_t> idx, part;
  std::vector<uint8_t> msig, mpk, mmode;
  for (uint64_t p : slow) {
    const hs_queue::req &r = q->reqs[p & q->mask];
    std::fill(q->wbits.begin(), q->wbits.begin() + (r.n + 31) / 32, 0u);
    int rc = HS_OK;
    if (r.msgs) {  // a preimage request: one hs_verify_groups call, the request as one group with per-item modes
      msig.resize((size_t)r.n * 64);
      mpk.resize((size_t)r.n * 32);
      mmode.resize(r.n);
      idx.assign(r.n, 0);  // group_idx
      for (uint32_t i = 0; i < r.n; i++) {
        const uint32_t s = (uint32_t)((p + i) & q->mask);
        memcpy(&msig[(size_t)i * 64], q->ring.recs.h[s].sig, 64);
        memcpy(&mpk[(size_t)i * 32], q->pk.h + 32 * (size_t)s, 32);
        mmode[i] = q->modes[s];
      }
      const uint8_t *a = q->arena_buf.h + r.a_off;
      uint32_t group_bit = 0;
      rc = hs_verify_groups(c, a + qmsg_o_pre(r.m, r.n), reinterpret_cast<const uint64_t *>(a), r.m, msig.data(), mpk.data(), nullptr,
                            reinterpret_cast<const uint32_t *>(a + 8 * ((size_t)r.m + 1)), idx.data(), mmode.data(), r.n, 1, q->wbits.data(), &group_bit);
    }
    for (uint32_t mode = HS_MODE_STRICT; mode <= HS_MODE_BATCH_EQ && rc == HS_OK && !r.msgs; mode++) {
      recs.clear();
      idx.clear();
      for (uint32_t i = 0; i < r.n; i++) {
        const uint32_t s = (uint32_t)((p + i) & q->mask);
        if (q->modes[s] != mode) continue;
        hs_rec128 x;
        memcpy(x.sig, q->ring.recs.h[s].sig, 64);
        memcpy(x.pk, q->pk.h + 32 * (size_t)s, 32);
        memcpy(x.msg, q->ring.recs.h[s].msg, 32);
        recs.push_back(x);
        idx.push_back(i);
      }
      if (recs.empty()) continue;
      part.assign((recs.size() + 31) / 32, 0);
      rc = hs_verify_rec128(c, recs.data(), recs.size(), mode, part.data());
      for (size_t k = 0; k < idx.size(); k++)
        if ((part[k >> 5] >> (k & 31)) & 1u) q->wbits[idx[k] >> 5] |= 1u << (idx[k] & 31);
    }
    {
      std::lock_guard<std::mutex> g(q->mu);
      queue_finish_locked(q, p, rc == HS_OK ? HS_OK : HS_ERR_CUDA, q->wbits.data(), fire);
    }
    queue_fire(fire);
  }
}

// One pass over the launches in flight: a device request whose completion word carries its launch's number is finished with
// its verdicts (the flags -> bits mapping of run_small).  A launch is retired once every request in its range — riders
// included — has its word.  Every 4,096 passes both streams are queried: a CUDA error, or a drained stream with a word still
// missing in a launch it ran, finishes the open requests with HS_ERR_CUDA (never an accept) and retires the launch.
static std::array<side_lane *, 2> queue_lanes(hs_queue *q);
static void lane_watch(hs_queue *q, side_lane &L, bool query);
static void queue_watch(hs_queue *q) {
  std::vector<queue_completion> fire;
  cudaError_t qes[2] = {cudaErrorNotReady, cudaErrorNotReady};  // [0] stream, [1] bulk_stream: a launch is judged by its own
  const bool query = (++q->spins & 0xfff) == 0;
  for (side_lane *L : queue_lanes(q)) lane_watch(q, *L, query);
  if (query) {  // queried BEFORE the words are read
    qes[0] = cudaStreamQuery(q->stream);
    qes[1] = cudaStreamQuery(q->bulk_stream);
  }
  for (cudaError_t x : qes)
    if (x != cudaSuccess && x != cudaErrorNotReady) fail(q->c, HS_ERR_CUDA, "verify queue kernel", x);
  {
    std::lock_guard<std::mutex> g(q->mu);
    for (size_t k = 0; k < q->inflight.size(); k++) {
      const hs_queue::launch L = q->inflight[k];
      const cudaError_t qe = qes[L.bulk ? 1 : 0];
      bool open = false;
      for (uint64_t p = L.lo; p < L.hi; p += q->reqs[p & q->mask].n) {
        hs_queue::req &r = q->reqs[p & q->mask];
        if (L.generic && !(r.gen && r.seq == L.seq)) continue;  // a request of another launch between its generic requests
        const bool mine = r.seq == L.seq && !r.finished;
        if (((volatile uint32_t *)q->ring.done.h)[p & q->mask] == L.seq) {
          if (!mine) continue;
          std::atomic_thread_fence(std::memory_order_acquire);
          uint32_t *bits = q->wbits.data();
          std::fill(bits, bits + (r.n + 31) / 32, 0u);
          for (uint32_t i = 0; i < r.n; i++) {  // the kernel writes both flags: each record's mode picks its verdict
            const uint32_t s = (uint32_t)((p + i) & q->mask);
            if (((volatile uint8_t *)q->ring.flags.h)[s] & mode_flag(q->modes[s])) bits[i >> 5] |= 1u << (i & 31);
          }
          if (L.sig_gen) {  // the completing block moved the request's signature-cache counts here before its completion word
            const volatile uint32_t *sc = q->sigc.hctr.h + HS_SIG_CTRS * (size_t)(p & q->mask);
            for (int k = 0; k < HS_SIG_CTRS; k++) q->sstats[k] += sc[k];
            if (L.sig_gen == q->sig_gen) q->sstats[4] += sc[2] - sc[3];
          }
          queue_finish_locked(q, p, HS_OK, bits, fire);
        } else if (qe == cudaErrorNotReady) {
          open = true;
        } else if (mine) {
          if (qe == cudaSuccess)
            fail(q->c, HS_ERR_CUDA, L.generic ? "verify queue: k_queue_generic did not complete"
                                    : L.bulk  ? "verify queue: k_verify_bulk did not complete"
                                              : "verify queue: k_verify_small did not complete");
          queue_finish_locked(q, p, HS_ERR_CUDA, nullptr, fire);
        }
      }
      if (!open) {
        q->inflight.erase(q->inflight.begin() + (long)k--);
        queue_release_locked(q);
      }
    }
  }
  queue_fire(fire);
}

// ---- side lanes (see lane_kind): what both lanes share
static std::array<side_lane *, 2> queue_lanes(hs_queue *q) { return {&q->batch, &q->explain}; }
// The first lane, in dispatch order, with no launch in flight and a ready request at the front of its list (null: none).
static side_lane *lane_ready_locked(hs_queue *q) {
  for (side_lane *L : queue_lanes(q))
    if (L->launch.empty() && !L->reqs.empty() && L->reqs.front().ready) return L;
  return nullptr;
}
// Waits for L's last launch: its buffers may be released after this.
static cudaError_t lane_drain(const side_lane &L) {
  const cudaError_t e = L.buf.stream ? cudaStreamSynchronize(L.buf.stream) : cudaSuccess;
  const cudaError_t f = L.buf.side ? cudaStreamSynchronize(L.buf.side) : cudaSuccess;
  return e != cudaSuccess ? e : f;
}

// Completes each open request of L's launch whose completion word carries the launch's number.  qe is what the lane's streams report:
// cudaErrorNotReady leaves the others open; drained streams (cudaSuccess) or an error (a failed enqueue passes cudaErrorLaunchFailure)
// complete them with HS_ERR_CUDA (never a result).  Once none is open, the launch is counted when every request of it completed HS_OK
// and its regions are released; its requests leave L's list only after their callbacks ran, so a resize returns after them.
static void lane_complete(hs_queue *q, side_lane &L, cudaError_t qe) {
  std::vector<queue_completion> fire;
  bool open = false, ok = true;
  {
    std::lock_guard<std::mutex> g(q->mu);
    for (lane_req *r : L.launch) {
      if (r->done) continue;
      const uint8_t *a = L.buf.arena.h + r->a_off;
      if (reinterpret_cast<const volatile uint32_t *>(a + r->o_tail)[1] == r->seq) {
        std::atomic_thread_fence(std::memory_order_acquire);
        ticket_close_locked(q, r->sink, HS_OK, r->n_bits, reinterpret_cast<const uint32_t *>(a + r->o_res), fire);
      } else if (qe == cudaErrorNotReady) {
        open = true;
        continue;
      } else {
        if (qe == cudaSuccess) fail(q->c, HS_ERR_CUDA, L.kind.incomplete);
        ticket_close_locked(q, r->sink, HS_ERR_CUDA, r->n_bits, nullptr, fire);
        ok = false;
      }
      r->done = true;
    }
    if (!open) {
      if (ok) L.kind.count(q, L);
      L.ring.release_to(L.launch.back()->a_end);
    }
  }
  queue_fire(fire);
  if (open) return;
  std::lock_guard<std::mutex> g(q->mu);
  L.reqs.erase(L.reqs.begin(), L.reqs.begin() + (long)L.launch.size());
  L.launch.clear();
  q->cv_done.notify_all();  // for callback tickets too: a resize waits for the lane's list to empty
}

// One launch takes the ready requests at the front of L's list, at most L.kind.per_launch of them, and enqueues its work under c->mu
// only while it enqueues.  A failed enqueue completes every request of the launch with HS_ERR_CUDA.
static void lane_dispatch(hs_queue *q, side_lane &L) {
  {
    std::lock_guard<std::mutex> g(q->mu);
    const uint32_t seq = ++L.seq ? L.seq : ++L.seq;  // never 0: the regions' tails were zeroed at submit
    for (size_t k = 0; k < L.reqs.size() && k < L.kind.per_launch && L.reqs[k].ready; k++) {
      L.reqs[k].seq = seq;
      L.launch.push_back(&L.reqs[k]);
    }
  }
  int rc;
  {
    std::lock_guard<std::mutex> g(q->c->mu);
    rc = L.kind.enqueue(q, L);
  }
  if (rc != HS_OK) lane_complete(q, L, cudaErrorLaunchFailure);
}

// Polls L's launch in flight.  When `query`, the lane's streams are queried first, before the words are read: a CUDA error fails the
// open requests, and drained streams with a word still missing mean the launch did not complete.
static void lane_watch(hs_queue *q, side_lane &L, bool query) {
  if (L.launch.empty()) return;  // (set and cleared on this thread)
  cudaError_t qe = cudaErrorNotReady;
  if (query) {
    const cudaError_t s[2] = {cudaStreamQuery(L.buf.stream), L.buf.side ? cudaStreamQuery(L.buf.side) : cudaSuccess};
    if (s[0] == cudaSuccess && s[1] == cudaSuccess) qe = cudaSuccess;
    for (cudaError_t x : s)
      if (x != cudaSuccess && x != cudaErrorNotReady) {
        fail(q->c, HS_ERR_CUDA, L.kind.launch_err, x);
        qe = x;
      }
  }
  lane_complete(q, L, qe);
}

// Resizes lane L to max_recs records and max_bytes bytes per request, or turns it off (0, 0).  It refuses new requests, waits for the
// submitted ones to complete and for the lane's streams to drain (a failed drain is HS_ERR_CUDA and leaves the lane off), and releases
// the lane's buffers and its own scratch before it allocates new ones: an arena where two of the largest regions fit (one can be
// filled while the other's launch runs), its mirror, a stream at the device's lowest priority, and what own(scratch, buffers, arena
// bytes, the device's highest stream priority) allocates.
template <class Scratch, class Own>
static int lane_configure(hs_queue *q, side_lane &L, size_t max_recs, size_t max_bytes, Scratch &scr, Own own) {
  hs_ctx *c = q->c;
  std::lock_guard<std::mutex> cfg(L.cfg_mu);
  {
    std::unique_lock<std::mutex> lk(q->mu);
    if (max_recs == L.max_recs && max_bytes == L.max_bytes) return HS_OK;
    L.max_recs = L.max_bytes = 0;  // refuses new requests while the lane changes
    q->cv_done.wait(lk, [&] { return L.reqs.empty(); });
  }
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, lane_drain(L));
  L.buf = {};  // released before the new lane is allocated
  scr = {};
  L.ring = byte_ring{};
  if (!max_recs) return HS_OK;
  uint64_t acap = 4096;
  while (acap < 2 * (uint64_t)max_bytes) acap <<= 1;
  lane_bufs B;
  Scratch S;
  int lo = 0, hi = 0;
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (e == cudaSuccess) e = create(B.stream, lo);
  if (e == cudaSuccess) e = alloc(B.arena, acap);
  if (e == cudaSuccess) e = alloc(B.mirror, acap);
  if (e == cudaSuccess) e = own(S, B, acap, hi);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(c, HS_ERR_NOMEM, (std::string(L.kind.configure) + ": no pinned host or device memory for the " + L.kind.name + " lane").c_str(), e);
  }
  memset(B.arena.h, 0, acap);
  L.buf = std::move(B);
  scr = std::move(S);
  std::lock_guard<std::mutex> g(q->mu);
  L.ring = byte_ring{acap, 0, 0};
  L.max_recs = max_recs;
  L.max_bytes = max_bytes;
  return HS_OK;
}

// ---- batch lane (hs_queue_submit_batch): one hs_verify_groups pass per request, on the lane's streams and scratch
// A request's region: pre_off (u64, n_msgs + 1) | preimages | sig (64 B each) | pk (32 B each) | msg_idx (u32) | group_idx (u32) |
// modes (u8) | result words (group words, then item words) | tail: [0] items outside the committee, [1] completion word.  Every
// section starts 16-byte aligned.  The inputs (everything before the result words) cross the bus in one copy into the mirror.
struct batch_layout {
  uint64_t o_pre, o_sig, o_pk, o_mi, o_gi, o_mo, o_res, o_tail, size;
};
static batch_layout batch_layout_of(uint64_t n_msgs, uint64_t pre_bytes, uint64_t n, uint64_t n_groups) {
  auto al = [](uint64_t x) { return (x + 15) & ~(uint64_t)15; };
  batch_layout b;
  b.o_pre = al(8 * (n_msgs + 1));
  b.o_sig = b.o_pre + al(pre_bytes);
  b.o_pk = b.o_sig + 64 * n;
  b.o_mi = b.o_pk + 32 * n;
  b.o_gi = b.o_mi + al(4 * n);
  b.o_mo = b.o_gi + al(4 * n);
  b.o_res = b.o_mo + al(n);
  b.o_tail = b.o_res + al(4 * ((n_groups + 31) / 32 + (n + 31) / 32));
  b.size = b.o_tail + 16;
  return b;
}
// A batch ticket's verdict bits: whole words, the group words then the item words.
static uint32_t batch_bits(uint64_t n_groups, uint64_t n) { return (uint32_t)(32 * ((n_groups + 31) / 32 + (n + 31) / 32)); }

// Enqueues the pass of the launch's one request.  Touches no scratch, stream, event or per-call state of the context, so synchronous
// calls, `_dev` calls and the queue's other launches can be in flight meanwhile.
static int batch_enqueue(hs_queue *q, side_lane &L) {
  hs_ctx *c = q->c;
  lane_req &r = *L.launch.front();
  const batch_layout B = batch_layout_of(r.m, r.pre_bytes, r.n, r.n_groups);
  batch_scratch &S = q->batch_scr;
  cudaStream_t s = L.buf.stream;
  const uint8_t *m = L.buf.mirror + r.a_off;
  HS_CUDA(c, cudaMemcpyAsync(L.buf.mirror + r.a_off, L.buf.arena.h + r.a_off, B.o_res, cudaMemcpyHostToDevice, s));
  k_digest32<<<blocks_for(r.m), HS_THREADS, 0, s>>>(m + B.o_pre, reinterpret_cast<const uint64_t *>(m), 0, r.m, S.dig);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  in_layout I{m + B.o_sig, 64, m + B.o_pk, 32, nullptr, reinterpret_cast<const uint8_t *>(S.dig.get()), 32, reinterpret_cast<const uint32_t *>(m + B.o_mi),
              nullptr, 32, 0};
  // only an explicitly registered committee: learned key-cache tables may be rebuilt by a synchronous call, and the lane never learns
  const bool committee = committee_registered(c);
  const pass_scratch P{S.xyz, S.meta, S.vidx, S.miss, S.miss_count, L.buf.side, {S.ev[0], S.ev[1]}, nullptr};
  // the queue shares its signature cache (hs_queue_sig_share): the pass probes and fills it
  const bool share = committee && c->share_q == q && q->d_sig;
  const share_pass SH{sig_cache_dev{q->d_sig, q->sigc.key, q->sig_bmask, S.share_ctr, nullptr}, S.share_list, S.share_fl, S.share_h.h};
  r.share_gen = share ? q->sig_gen : 0;
  HS_TRY(launch_main(c, I, r.n, committee, false, ctx_tables(c), P, s, [](bool) { return HS_OK; }, share ? &SH : nullptr));
  const int fin_group = r.n >= (1u << 19) ? 16 : (r.n >= (1u << 18) ? 8 : 4);
  HS_TRY(launch_finish(c, I, r.n, S.xyz, S.meta, HS_MODE_STRICT, m + B.o_mo, S.items, peer_route{}, fin_group, s, share ? &SH : nullptr));
  if (share) {
    HS_TRY(launch_sig_fill(c, I, r.n, ctx_tables(c).C, SH, S.meta, HS_MODE_STRICT, m + B.o_mo, s));
    HS_CUDA(c, cudaEventRecord(q->ev_share, s));
  }
  HS_CUDA(c, cudaMemsetAsync(S.grej, 0, 4 * ((r.n_groups + 31) / 32), s));
  uint8_t *res = L.buf.arena.d + r.a_off;
  k_batch_done<<<blocks_for(r.n, 256), 256, 0, s>>>(S.items, reinterpret_cast<const uint32_t *>(m + B.o_gi), r.n, r.n_groups, S.grej,
                                                    reinterpret_cast<uint32_t *>(res + B.o_res), committee ? S.miss_count.get() : nullptr,
                                                    reinterpret_cast<uint32_t *>(res + B.o_tail), r.seq, S.counter);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
static void batch_count(hs_queue *q, side_lane &L) {
  for (const lane_req *r : L.launch) {
    if (r->share_gen) sig_share_count(q, q->batch_scr.share_h.h, r->share_gen);
    L.stats[0]++;
    L.stats[1] += r->n;
    L.stats[2] += r->n_groups;
    L.stats[3] += r->pre_bytes;
    L.stats[4] += reinterpret_cast<const volatile uint32_t *>(L.buf.arena.h + r->a_off + r->o_tail)[0];
  }
}

// ---- explain lane (hs_queue_submit_explain, hs_queue_submit_explain_msgs): k_queue_explain over every ready request, on the lane's stream
// An explain ticket's bits: the why bytes packed four to a word, little-endian.
static uint32_t explain_bits(uint64_t n) { return (uint32_t)(32 * ((n + 3) / 4)); }
// The launch's regions are one span of arena positions, which crosses the bus in at most two copies (the span may wrap once) into the
// mirror, tails included: k_queue_explain counts in the mirror's tails.  The launch reads no context table, so nothing else of the
// context waits for it.
static int explain_enqueue(hs_queue *q, side_lane &L) {
  hs_ctx *c = q->c;
  uint32_t recs = 0;
  for (size_t k = 0; k < L.launch.size(); k++) {
    const lane_req &r = *L.launch[k];
    q->explain_scr.list.h[k] = xq_desc{r.a_off, r.n, recs, r.m, (uint32_t)r.pre_bytes, r.seq, 0};
    recs += r.n;
  }
  cudaStream_t s = L.buf.stream;
  const uint64_t p0 = L.launch.front()->a_pos, p1 = L.launch.back()->a_end;
  const uint64_t o0 = L.ring.off(p0), first = std::min(p1 - p0, L.ring.cap - o0);
  cudaError_t e = cudaMemcpyAsync(L.buf.mirror + o0, L.buf.arena.h + o0, first, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess && p1 - p0 > first) e = cudaMemcpyAsync(L.buf.mirror.get(), L.buf.arena.h, p1 - p0 - first, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = launch_queue_explain(c, q->explain_scr.list.d, (uint32_t)L.launch.size(), recs, L.buf.mirror, L.buf.arena.d, s);
  return e == cudaSuccess ? HS_OK : fail(c, HS_ERR_CUDA, "verify queue explain launch", e);
}
static void explain_count(hs_queue *, side_lane &L) {
  L.stats[0]++;
  for (const lane_req *r : L.launch) L.stats[1] += r->n;
  L.stats[2] += L.launch.size();
}

static size_t queue_small_inflight_locked(const hs_queue *q) {
  size_t k = 0;
  for (const hs_queue::launch &L : q->inflight) k += !L.bulk;
  return k;
}
// Generic requests wait in gpend and no generic launch is in flight (or the option is off: they take the slow path).
static bool queue_generic_ready_locked(const hs_queue *q) {
  if (q->gpend.empty()) return false;
  if (!q->gen_on.load()) return true;
  for (const hs_queue::launch &L : q->inflight)
    if (L.generic) return false;
  return true;
}

static void queue_main(hs_queue *q) {
  cudaSetDevice(q->c->device);
  t_queue_dispatcher = true;
  const std::array<side_lane *, 2> lanes = queue_lanes(q);
  std::unique_lock<std::mutex> lk(q->mu);
  for (;;) {
    if (!q->cc_ready.empty()) {  // requests the certificate cache answered at submit
      std::vector<cert_req *> ready;
      ready.swap(q->cc_ready);
      std::vector<queue_completion> fire;
      for (cert_req *cr : ready) cert_complete_locked(q, cr, fire);
      lk.unlock();
      queue_fire(fire);
      lk.lock();
    } else if (side_lane *L = lane_ready_locked(q)) {  // first: one short enqueue, and a vote burst would otherwise keep postponing it
      lk.unlock();
      lane_dispatch(q, *L);
      lk.lock();
    } else if ((q->launched < q->tail && queue_small_inflight_locked(q) < HS_QUEUE_MAX_INFLIGHT) || queue_generic_ready_locked(q)) {
      // everything pending; only the waiting generic requests while the small launches are at their limit
      const uint64_t lo = q->launched, hi = queue_small_inflight_locked(q) < HS_QUEUE_MAX_INFLIGHT ? q->tail : lo;
      q->launched = hi;
      lk.unlock();
      queue_dispatch(q, lo, hi);
      lk.lock();
    } else if (!q->inflight.empty() || std::any_of(lanes.begin(), lanes.end(), [](side_lane *L) { return !L->launch.empty(); })) {
      lk.unlock();
      queue_watch(q);
      lk.lock();
    } else if (q->stop && std::all_of(lanes.begin(), lanes.end(), [](side_lane *L) { return L->reqs.empty(); })) {
      // (a lane request still being copied in is announced on cv_work)
      break;
    } else {
      q->cv_work.wait(lk);
    }
  }
}

static void queue_free(hs_queue *q) {
  {
    std::lock_guard<std::mutex> g(q->mu);
    q->stop = true;
  }
  q->cv_work.notify_all();
  if (q->th.joinable()) q->th.join();  // the thread finishes every request first
  cudaSetDevice(q->c->device);
  // the last launches' blocks have exited before the ring goes
  if (q->ev_last) cudaEventSynchronize(q->ev_last);
  if (q->ev_bulk_last) cudaEventSynchronize(q->ev_bulk_last);
  if (q->ev_audit) cudaEventSynchronize(q->ev_audit);
  for (side_lane *L : queue_lanes(q)) lane_drain(*L);
  delete q;  // the owners release the rest
}

// Digest of n fixed-size messages: staged/coalesced kernel when every message starts 16-byte aligned and has at least one
// full block, the generic per-thread reader otherwise.
static int launch_digest_fixed(hs_ctx *c, const uint8_t *d_msgs, size_t msg_len, size_t n, uint32_t *d_out, cudaStream_t stream) {
  if (msg_len >= 128 && (msg_len & 15) == 0 && (reinterpret_cast<uintptr_t>(d_msgs) & 15) == 0) {
    sha512_kw kw;
    const int pad_is_const = (msg_len & 127) == 0;
    if (pad_is_const) sha512_pad_schedule(kw, msg_len);
    else memset(&kw, 0, sizeof(kw));
    k_digest32_fixed<<<blocks_for(n), HS_THREADS, 0, stream>>>(d_msgs, msg_len, n, d_out, kw, pad_is_const);
  } else {
    k_digest32<<<blocks_for(n), HS_THREADS, 0, stream>>>(d_msgs, nullptr, msg_len, n, d_out);
  }
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
// Digest of a few long messages: one warp per message, schedules expanded in parallel across lanes.
static int launch_digest_long(hs_ctx *c, const uint8_t *d_data, const uint64_t *d_off, size_t n, uint32_t *d_out, cudaStream_t stream) {
  k_digest32_long<<<(unsigned)n, 32, 0, stream>>>(d_data, d_off, n, d_out);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}

// off[0] == 0 and off[i] <= off[i+1]: a decreasing offset would make a length wrap to ~2^64 on the device
static bool offsets_ok(const uint64_t *off, size_t n) {
  if (off[0] != 0) return false;
  for (size_t i = 0; i < n; i++)
    if (off[i] > off[i + 1]) return false;
  return true;
}
static in_layout layout_rec128(const void *d_recs) {
  const uint8_t *r = (const uint8_t *)d_recs;
  return in_layout{r, 128, r + 64, 128, nullptr, r + 96, 128, nullptr, nullptr, 32, 1};
}

// ---- argument checks shared with the multi-device context (hs_args.h)
const char *hs_args::rec128(const hs_rec128 *recs, size_t n, uint32_t mode, const uint32_t *out_bitmap) {
  return (mode > 1 || (n && (!recs || !out_bitmap))) ? "bad argument" : nullptr;
}
const char *hs_args::msgs(const uint8_t *sig, const uint8_t *pk, const uint32_t *vidx, const uint8_t *msgs, size_t msg_len, size_t n, uint32_t mode,
                          const uint32_t *out_bitmap) {
  return (mode > 1 || (n && (!sig || (!pk && !vidx) || !msgs || !out_bitmap || msg_len == 0))) ? "bad argument" : nullptr;
}
const char *hs_args::groups(const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                            const uint32_t *vidx, const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *mode, size_t n_items,
                            size_t n_groups, const uint32_t *out_group_bitmap) {
  if (!out_group_bitmap || (n_msgs && !pre_off) || (n_items && (!sig || !msg_idx || !group_idx || (!pk && !vidx) || n_msgs == 0 || n_groups == 0)))
    return "bad argument";
  if (n_items && (!offsets_ok(pre_off, n_msgs) || (pre_off[n_msgs] && !preimages))) return "bad preimage offsets";
  for (size_t i = 0; i < n_items; i++)
    if (msg_idx[i] >= n_msgs || group_idx[i] >= n_groups || (mode && mode[i] > 1)) return "index out of range";
  return nullptr;
}
// HS_ERR_ARG with "<entry point>: <reason>" when a shared check above refuses the call
static int fail_args(hs_ctx *c, const char *entry, const char *why) { return fail(c, HS_ERR_ARG, (std::string(entry) + ": " + why).c_str()); }

extern "C" {

int hs_ctx_create(hs_ctx **out, int device, uint32_t flags) {
  if (!out) return HS_ERR_ARG;
  int wb = (int)(flags & 0xffu);
  if (wb == 0) wb = 24;  // 11 windows x 2^23 entries x 96 B = 8.9 GB of HBM for 11 instead of 16+ additions per [S]B
  if (wb < 8 || wb > 26 || (wb % 2)) return HS_ERR_ARG;  // 26 bits: 10 windows, 32 GB — one addition fewer per verify than the 8.9 GB default
  *out = nullptr;
  hs_ctx *c = new (std::nothrow) hs_ctx();
  if (!c) return HS_ERR_NOMEM;
  c->device = device;
  cudaError_t e = cudaSetDevice(device);
  int sms = 0;
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  c->n_sms = (unsigned)sms;
  if (e == cudaSuccess) e = create(c->stream);
  if (e == cudaSuccess) e = create(c->stream2);
  if (e == cudaSuccess) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    e = create(c->stream_side, hi);
  }
  for (int i = 0; i < 2 && e == cudaSuccess; i++) {
    e = create(c->ev[i]);
    if (e == cudaSuccess) e = create(c->ev_done[i]);
    if (e == cudaSuccess) e = create(c->ev_side[i]);
  }
  if (e == cudaSuccess) e = create(c->ev_dev_pass);
  if (e == cudaSuccess) e = alloc(c->d_miss_count, 4);
  if (e == cudaSuccess) e = create(c->stream_tail);
  if (e == cudaSuccess) e = create(c->ev_main_done);
  if (e == cudaSuccess) e = create(c->ev_results);
  for (int i = 0; i < 2 && e == cudaSuccess; i++) e = create(c->ev_tail[i]);
  if (e == cudaSuccess) e = make_ring(c->small, HS_SMALL_MAX, c->stream);
  c->small_enabled = !(getenv("HS_SMALL_PATH") && getenv("HS_SMALL_PATH")[0] == '0');
  set_window(c->cp, false, wb);
  set_window(c->cp, true, 12);
  c->wa_forced = (int)((flags >> 8) & 0xffu);
  if (const char *b = getenv("HS_TABLE_BUDGET_MB")) c->table_budget = (size_t)strtoull(b, nullptr, 10) << 20;
  c->cache_wanted = c->cache_enabled = !(flags & HS_FLAG_NO_KEY_CACHE) && !(getenv("HS_KEY_CACHE") && getenv("HS_KEY_CACHE")[0] == '0');
  if (e == cudaSuccess) e = alloc(c->d_btable, sizeof(ge_niels) * comb_table_entries(wb));
  if (e == cudaSuccess) {
    if (launch_build(c, nullptr, nullptr, 1, 0, wb, c->cp.nb, c->d_btable, nullptr, c->stream) != HS_OK) e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) {
    fprintf(stderr, "hs_ctx_create: CUDA failure: %s\n", cudaGetErrorString(e));
    hs_ctx_destroy(c);
    return HS_ERR_CUDA;
  }
  *out = c;
  return HS_OK;
}

void hs_ctx_destroy(hs_ctx *c) {
  if (!c) return;
  hs_scrub_stop(c);  // joins the scrub's thread before anything it uses goes
  std::vector<hs_queue *> qs;
  {
    std::lock_guard<std::mutex> g(c->queues_mu);
    qs.swap(c->queues);
  }
  for (hs_queue *q : qs) queue_free(q);  // completes their requests (callbacks fire) and joins their threads
  { std::lock_guard<std::mutex> a(c->audit_mu); }  // an audit still waiting on its kernels returns before its tables go
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  delete c;  // the owners release the rest
}

const char *hs_last_error(const hs_ctx *c) { return c ? c->err.c_str() : "null context"; }
size_t hs_cached_keys(const hs_ctx *c) { return (c && !c->explicit_committee) ? c->n_keys : 0; }
void hs_window_bits(const hs_ctx *c, int *key_bits, int *base_bits) {
  if (key_bits) *key_bits = (c && has_key_tables(c)) ? c->cp.wa : 0;
  if (base_bits) *base_bits = c ? c->cp.wb : 0;
}
uint64_t hs_kernel_launches(const hs_ctx *c) { return c ? c->launches.load() : 0; }
/* Measurement hook: with profiling on, CUDA events bracket the k_verify_main<committee> launch of every verify pass on the stream the
 * pass runs on; hs_profile_main_ms() waits for the last pass and returns that kernel's duration in ms (< 0: nothing recorded). */
/* Deferred-results mode for streams of `_dev` verify passes: the tail of a pass (finish kernel + peer exchange, hs_qc_and_dev) runs on an
 * internal stream and overlaps the NEXT pass's kernels; verdict bitmaps are complete only after hs_results_wait(ctx, stream) (which makes
 * `stream` wait for every tail enqueued so far).  Inputs of a pass (signatures) must stay valid until then.  Host-pointer entry points are
 * unaffected: switch the mode only while no pass is in flight. */
int hs_set_deferred(hs_ctx *c, int on) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaDeviceSynchronize());
  c->deferred = on != 0;
  c->flip = 0;
  return HS_OK;
}
int hs_results_wait(hs_ctx *c, void *stream) {
  if (!c) return HS_ERR_ARG;
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaEventRecord(c->ev_results, c->stream_tail));
  HS_CUDA(c, cudaStreamWaitEvent((cudaStream_t)stream, c->ev_results, 0));
  return HS_OK;
}
int hs_profile_enable(hs_ctx *c, int on) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  for (int i = 0; i < 2 && on; i++)
    if (!c->ev_prof[i]) HS_CUDA(c, create(c->ev_prof[i], cudaEventDefault));
  c->profile_main = on != 0;
  return HS_OK;
}
double hs_profile_main_ms(hs_ctx *c) {
  if (!c || !c->ev_prof[1]) return -1.0;
  cudaSetDevice(c->device);
  if (cudaEventSynchronize(c->ev_prof[1]) != cudaSuccess) return -1.0;
  float ms = -1.0f;
  if (cudaEventElapsedTime(&ms, c->ev_prof[0], c->ev_prof[1]) != cudaSuccess) return -1.0;
  return (double)ms;
}

void *hs_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void hs_host_free(void *p) {
  if (p) cudaFreeHost(p);
}

// ---- committee registration
// Bytes the per-key tables of a registration may take now: ~62 % of the device by default (80 GB H100: 16 bits up to ~1 k keys, 15
// up to ~1.8 k, 14 up to ~3.3 k, 13 up to ~6.3 k, 12 up to ~11 k), or HS_TABLE_BUDGET_MB / hs_set_table_budget for a shared device,
// and never more than 7/8 of the free memory.
static int committee_budget(hs_ctx *c, size_t &budget) {
  size_t free_b = 0, total_b = 0;
  HS_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
  budget = total_b / 100 * 62;
  if (c->table_budget) budget = c->table_budget;
  if (budget > free_b - free_b / 8) budget = free_b - free_b / 8;
  return HS_OK;
}
// Table slots of a committee of N keys: spare slots (1/16 of the set, at least 16) let hs_committee_update add validators without
// rebuilding anything.
static size_t committee_capacity(size_t N) { return N + (N / 16 > 16 ? N / 16 : 16); }
// Table slots (capk: N plus spares) and per-key window (wa) that registering N keys picks now: the widest window whose tables fit in
// the budget.
static int committee_geometry(hs_ctx *c, size_t N, size_t &capk, int &wa) {
  size_t budget = 0;
  HS_TRY(committee_budget(c, budget));
  capk = committee_capacity(N);
  wa = 8;
  for (int w : {17, 16, 15, 14, 13, 12, 11, 10, 9, 8}) {  // 17 bits: 15 windows (94 MB per key: committees up to ~500 keys on 80 GB); 18 would still need 15
    if (c->wa_forced && w != c->wa_forced) continue;
    wa = w;
    if (capk * comb_table_entries(w) * sizeof(ge_niels) <= budget) break;
  }
  return HS_OK;
}
static int committee_register_locked(hs_ctx *c, const uint8_t *pks, size_t N, uint32_t *out_valid_bitmap) {
  HS_CUDA(c, cudaSetDevice(c->device));
  // Drains every stream of the device, the verify queues' included: a queue enqueues a launch only while it holds c->mu, so
  // nothing launched against the old tables survives this line, and later dispatches resolve keys against the new mirror.
  HS_CUDA(c, cudaDeviceSynchronize());
  cache_release(c);
  c->learn_pending = false;
  c->cache_full = false;
  c->explicit_committee = false;   // set only once the new tables are complete: a failed registration leaves NO committee
  c->cache_enabled = c->cache_wanted;
  if (N == 0) return HS_OK;        // clears the committee and hands key handling back to the cache (if enabled)
  size_t capk = 0;
  int wa = 8;
  HS_TRY(committee_geometry(c, N, capk, wa));
  key_index index;
  index.reset(capk);
  index.build(pks, N, [](size_t) { return true; });
  if (sc_ndigits_rt(wa) + c->cp.nb > HS_MAX_DIGITS) return fail(c, HS_ERR_ARG, "window combination exceeds HS_MAX_DIGITS");
  cudaError_t e = make_key_store(c->keys, capk, index.slots.size(), wa, c->stream);  // the old tables were released above
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(c, HS_ERR_NOMEM, "committee tables do not fit in device memory", e);
  }
  set_window(c->cp, true, wa);
  c->a_table_entries = comb_table_entries(wa);
  int rc = HS_OK;
  e = cudaMemcpyAsync(c->keys.pks, pks, N * 32, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(c->keys.slots, index.slots.data(), index.slots.size() * 4, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) rc = launch_build(c, c->keys.pks, nullptr, N, 1, wa, c->cp.na, c->keys.atables, c->keys.key_flags, c->stream);
  if (e == cudaSuccess && rc == HS_OK) e = cudaStreamSynchronize(c->stream);
  std::vector<uint8_t> fl(N);
  if (e == cudaSuccess && rc == HS_OK) e = cudaMemcpy(fl.data(), c->keys.key_flags, N, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess || rc != HS_OK) {
    cache_release(c);
    return rc != HS_OK ? rc : fail(c, HS_ERR_CUDA, "committee registration", e);
  }
  c->n_keys = N;
  c->key_capacity = capk;
  c->explicit_committee = true;
  c->h_pks.assign(pks, pks + N * 32);  // host mirror: hs_committee_update edits the set incrementally
  c->h_index = std::move(index);
  c->h_key_live.assign(N, 1);
  if (out_valid_bitmap) {
    for (size_t w = 0; w < (N + 31) / 32; w++) out_valid_bitmap[w] = 0;
    for (size_t i = 0; i < N; i++)
      if (fl[i] & 1) out_valid_bitmap[i >> 5] |= 1u << (i & 31);
  }
  return HS_OK;
}
int hs_committee_register(hs_ctx *c, const uint8_t *pks, size_t N, uint32_t *out_valid_bitmap) {
  if (!c || (N && !pks) || N >= HS_NO_KEY) return fail(c, HS_ERR_ARG, "hs_committee_register: bad argument");
  std::lock_guard<std::mutex> g(c->mu);
  return committee_register_locked(c, pks, N, out_valid_bitmap);
}

// Rebuilds the open-addressing table from the host mirror (deletions leave no tombstones; the first of duplicated key bytes wins) over
// the slots in service: every learned key of the key cache, a committee's live slots but those under repair (SLOT_REPAIR).  Publishes
// it on the context's stream and waits, so that every launch enqueued afterwards, on any stream, probes the new table.
static int publish_hash(hs_ctx *c) {
  c->h_index.build(c->h_pks.data(), c->n_keys, [c](size_t i) { return !c->explicit_committee || c->h_key_live[i] == SLOT_LIVE; });
  HS_CUDA(c, cudaMemcpyAsync(c->keys.slots, c->h_index.slots.data(), c->h_index.slots.size() * 4, cudaMemcpyHostToDevice, c->stream));
  HS_CUDA(c, cudaStreamSynchronize(c->stream));
  return HS_OK;
}

// The slots hs_committee_update gives added keys, chosen on copies of the mirrors: a key in service keeps its index, the same key twice
// takes one slot, a new key takes the lowest free slot, then a spare.  Each slot taken is marked `mark` in `live`.  full: no slot was
// left for key idx.size(), and the keys before it are planned.
struct slot_plan {
  std::vector<uint8_t> live, pks;  // h_key_live and h_pks with the additions (longer by the spares taken)
  std::vector<uint32_t> idx;       // the index of each added key
  std::vector<uint32_t> fresh;     // the slots taken, in order
  bool full = false;
};
static void plan_adds(const hs_ctx *c, const uint8_t *add_pks, size_t n_add, uint8_t mark, slot_plan &P) {
  P.live = c->h_key_live;
  P.pks = c->h_pks;
  // The published table plus this call's additions, so that the same key twice in one call takes one slot.
  key_index index = c->h_index;
  auto live = [&P](uint32_t idx) { return P.live[idx] != 0; };
  size_t next_free = 0;
  for (size_t i = 0; i < n_add; i++) {
    const uint8_t *key = add_pks + 32 * i;
    uint32_t idx = index.find(P.pks.data(), key, live);
    if (idx == HS_NO_KEY) {
      while (next_free < P.live.size() && P.live[next_free]) next_free++;
      if (next_free < P.live.size()) idx = (uint32_t)next_free;
      else if (P.live.size() < c->key_capacity) {
        idx = (uint32_t)P.live.size();
        P.live.push_back(0);
        P.pks.resize(P.live.size() * 32);
      } else {
        P.full = true;
        return;
      }
      memcpy(P.pks.data() + 32 * (size_t)idx, key, 32);
      P.live[idx] = mark;
      index.insert_absent(P.pks.data(), idx, live);
      P.fresh.push_back(idx);
    }
    P.idx.push_back(idx);
  }
}
// Frees a pending or in-progress stage's slots (hs_committee_update, hs_committee_discard, a failed stage): they go back to free, and
// the spares it took are no longer held.  After a commit nothing is SLOT_STAGED, so this only forgets the stage.
static void stage_drop(hs_ctx *c) {
  for (uint32_t s : c->stage.fresh)
    if (s < c->h_key_live.size() && c->h_key_live[s] == SLOT_STAGED) c->h_key_live[s] = 0;
  if (c->explicit_committee && c->h_key_live.size() > c->n_keys) c->h_key_live.resize(c->n_keys);
  c->stage = {};
}

// Incremental epoch change (consensus/src/config.rs Committee: a few validators join / leave): removed indices stop
// verifying (flag cleared, hash slot dropped), added keys take a free slot — a removed one or a spare — and only THEIR tables
// are built, in one k_build_comb launch; every other validator keeps its index and its table.  It discards a pending stage.
int hs_committee_update(hs_ctx *c, const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove, uint32_t *out_add_idx) {
  if (!c || (n_add && (!add_pks || !out_add_idx)) || (n_remove && !remove_idx)) return fail(c, HS_ERR_ARG, "hs_committee_update: bad argument");
  std::lock_guard<std::mutex> g(c->mu);
  if (!c->explicit_committee) return fail(c, HS_ERR_ARG, "hs_committee_update: no committee registered");
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaDeviceSynchronize());  // epoch boundary: nothing of the old set may be in flight (verify queue launches and audits included)
  for (size_t i = 0; i < n_remove; i++)
    if (remove_idx[i] >= c->n_keys) return fail(c, HS_ERR_ARG, "hs_committee_update: remove index out of range");
  stage_drop(c);
  c->key_gen++;
  c->map_gen++;
  for (size_t i = 0; i < n_remove; i++) {
    c->h_key_live[remove_idx[i]] = 0;
    HS_CUDA(c, cudaMemsetAsync(c->keys.key_flags + remove_idx[i], 0, 1, c->stream));
  }
  // A failed update leaves the context's index as published; the keys planned before a lack of slots are still placed and built.
  slot_plan P;
  plan_adds(c, add_pks, n_add, SLOT_LIVE, P);
  c->h_key_live = std::move(P.live);
  c->h_pks = std::move(P.pks);
  c->n_keys = c->h_key_live.size();
  std::copy(P.idx.begin(), P.idx.end(), out_add_idx);
  const size_t n_new = P.fresh.size();
  if (n_new) {
    for (uint32_t s : P.fresh)
      HS_CUDA(c, cudaMemcpyAsync(c->keys.pks + 32 * (size_t)s, c->h_pks.data() + 32 * (size_t)s, 32, cudaMemcpyHostToDevice, c->stream));
    h2d_stage st;
    const size_t s_slots = st.add(P.fresh.data(), 4 * n_new), s_flags = st.add(nullptr, n_new);
    HS_TRY(st.upload(c, c->in[0], c->stream));
    HS_TRY(launch_build(c, c->keys.pks, reinterpret_cast<const uint32_t *>(st.ptr(s_slots)), n_new, 1, c->cp.wa, c->cp.na, c->keys.atables,
                        st.ptr(s_flags), c->stream));
    for (size_t k = 0; k < n_new; k++)
      HS_CUDA(c, cudaMemcpyAsync(c->keys.key_flags + P.fresh[k], st.ptr(s_flags) + k, 1, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (P.full) {
    HS_CUDA(c, cudaStreamSynchronize(c->stream));
    return fail(c, HS_ERR_NOMEM, "hs_committee_update: no free table slot (re-register the committee)");
  }
  HS_TRY(publish_hash(c));
  return HS_OK;
}
/* Upper bound (bytes) for the per-key tables of the NEXT registration / key-cache allocation; 0 = default (~62 % of the device). */
int hs_set_table_budget(hs_ctx *c, size_t bytes) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(c->mu);
  c->table_budget = bytes;
  return HS_OK;
}

// ---- device-resident entry points (one stream at a time per context: they share the context's scratch)
int hs_verify_rec128_dev(hs_ctx *c, const void *d_recs, size_t n, uint32_t mode, void *d_bitmap, void *stream) {
  if (!c || (n && (!d_recs || !d_bitmap)) || mode > 1) return fail(c, HS_ERR_ARG, "hs_verify_rec128_dev: bad argument");
  HS_CUDA(c, cudaSetDevice(c->device));
  return run_verify(c, layout_rec128(d_recs), n, mode, (uint32_t *)d_bitmap, (cudaStream_t)stream, false);
}
int hs_verify_var_dev(hs_ctx *c, const void *d_sig, const void *d_pk, const void *d_msgs, const void *d_off, size_t n, uint32_t mode,
                      void *d_bitmap, void *stream) {
  if (!c || mode > 1 || (n && (!d_sig || !d_pk || !d_off || !d_bitmap))) return fail(c, HS_ERR_ARG, "hs_verify_var_dev: bad argument");
  HS_CUDA(c, cudaSetDevice(c->device));
  in_layout L{(const uint8_t *)d_sig, 64, (const uint8_t *)d_pk, 32, nullptr, (const uint8_t *)d_msgs, 0, nullptr, (const uint64_t *)d_off, 0, 0};
  return run_verify(c, L, n, mode, (uint32_t *)d_bitmap, (cudaStream_t)stream, false);
}
int hs_verify_committee_dev(hs_ctx *c, const void *d_vidx, const void *d_sig, const void *d_midx, const void *d_digests, size_t n,
                            uint32_t mode, void *d_bitmap, void *stream) {
  if (!c || mode > 1 || (n && (!d_vidx || !d_sig || !d_digests || !d_bitmap))) return fail(c, HS_ERR_ARG, "hs_verify_committee_dev: bad argument");
  HS_CUDA(c, cudaSetDevice(c->device));
  // d_midx == NULL: every vote is over digests[0]
  in_layout L{(const uint8_t *)d_sig, 64, nullptr, 0, (const uint32_t *)d_vidx, (const uint8_t *)d_digests, d_midx ? (size_t)32 : (size_t)0,
              (const uint32_t *)d_midx, nullptr, 32, 0};
  return run_verify(c, L, n, mode, (uint32_t *)d_bitmap, (cudaStream_t)stream, true);
}
int hs_digest32_dev(hs_ctx *c, const void *d_data, const void *d_off, size_t n, void *d_out, void *stream) {
  if (!c || (n && (!d_off || !d_out))) return fail(c, HS_ERR_ARG, "hs_digest32_dev: bad argument");
  if (n == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  k_digest32<<<blocks_for(n), HS_THREADS, 0, (cudaStream_t)stream>>>((const uint8_t *)d_data, (const uint64_t *)d_off, 0, n, (uint32_t *)d_out);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
int hs_digest32_fixed_dev(hs_ctx *c, const void *d_msgs, size_t msg_len, size_t n, void *d_out, void *stream) {
  if (!c || (n && (!d_msgs || !d_out || msg_len == 0))) return fail(c, HS_ERR_ARG, "hs_digest32_fixed_dev: bad argument");
  if (n == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  return launch_digest_fixed(c, (const uint8_t *)d_msgs, msg_len, n, (uint32_t *)d_out, (cudaStream_t)stream);
}
int hs_verify_msgs_dev(hs_ctx *c, const void *d_sig, const void *d_pk, const void *d_vidx, const void *d_msgs, size_t msg_len, size_t n,
                       uint32_t mode, void *d_digests, void *d_bitmap, void *stream) {
  if (!c || mode > 1 || (n && (!d_sig || (!d_pk && !d_vidx) || !d_msgs || !d_digests || !d_bitmap)))
    return fail(c, HS_ERR_ARG, "hs_verify_msgs_dev: bad argument");
  if (n == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  // Digest(msg_i) in its own kernel: fused into k_verify_main, the SHA phase would run at the curve kernel's 128-register
  // occupancy, and the two phases do not overlap across pipes in practice.
  HS_TRY(launch_digest_fixed(c, (const uint8_t *)d_msgs, msg_len, n, (uint32_t *)d_digests, (cudaStream_t)stream));
  in_layout L{(const uint8_t *)d_sig, 64, (const uint8_t *)d_pk, 32, (const uint32_t *)d_vidx, (const uint8_t *)d_digests, 32, nullptr, nullptr, 32, 0};
  return run_verify(c, L, n, mode, (uint32_t *)d_bitmap, (cudaStream_t)stream, d_vidx != nullptr);
}

// ---- QC::verify for many certificates (consensus/src/messages.rs:180-208)
int hs_verify_qcs(hs_ctx *c, const uint8_t *preimages, size_t n_qc, const uint8_t *pk, const uint32_t *vidx, const uint8_t *sig,
                  const uint32_t *qc_idx, size_t n_votes, uint32_t *out_vote_bitmap, uint32_t *out_qc_bitmap) {
  if (!c || !out_qc_bitmap || (n_qc && !preimages) || (n_votes && (!sig || !qc_idx || (!pk && !vidx) || n_qc == 0)))
    return fail(c, HS_ERR_ARG, "hs_verify_qcs: bad argument");
  for (size_t i = 0; i < n_votes; i++)
    if (qc_idx[i] >= n_qc) return fail(c, HS_ERR_ARG, "hs_verify_qcs: qc_idx out of range");
  const size_t qc_words = (n_qc + 31) / 32, vote_words = (n_votes + 31) / 32;
  const std::vector<uint32_t> ones = bitmap_ones(n_qc);
  if (n_votes == 0) {
    std::copy(ones.begin(), ones.end(), out_qc_bitmap);
    return HS_OK;
  }
  std::lock_guard<std::mutex> g(c->mu);
  share_call sh(c);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_pre = S.add(preimages, n_qc * 40), s_dig = S.add(nullptr, n_qc * 32), s_sig = S.add(sig, n_votes * 64),
               s_key = S.add(pk ? (const void *)pk : (const void *)vidx, n_votes * (pk ? 32 : 4)), s_qi = S.add(qc_idx, n_votes * 4);
  HS_TRY(ensure(c, c->out, (vote_words + qc_words) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  uint32_t *d_votes = (uint32_t *)c->out.p.get(), *d_qc = d_votes + vote_words;
  const uint32_t *d_qi = (const uint32_t *)S.ptr(s_qi);
  HS_CUDA(c, cudaMemcpyAsync(d_qc, ones.data(), qc_words * 4, cudaMemcpyHostToDevice, c->stream));
  // QC::digest = SHA-512(hash || round_le)[..32] for every certificate (messages.rs:201-208)
  k_digest32<<<blocks_for(n_qc), HS_THREADS, 0, c->stream>>>(S.ptr(s_pre), nullptr, 40, n_qc, (uint32_t *)S.ptr(s_dig));
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  HS_TRY(hs_verify_qc_votes_dev(c, S.ptr(s_dig), pk ? S.ptr(s_key) : nullptr, pk ? nullptr : S.ptr(s_key), S.ptr(s_sig), d_qi, n_votes, d_votes,
                                c->stream));
  HS_TRY(launch_qc_and(c, d_votes, d_qi, n_votes, n_qc, d_qc, c->stream));
  return readback(c, {{out_vote_bitmap, d_votes, vote_words * 4}, {out_qc_bitmap, d_qc, qc_words * 4}});
}

// ---- device-resident QC verification (strong-scaling path of BASELINE config[3]: the votes of many QCs sharded over ranks)
// Per-vote verdicts of this rank's shard (batch-eq condition).  d_qc_digests: n_qc x 32 (hs_digest32_fixed_dev over the 40-byte
// preimages); d_qc_idx selects each vote's digest.  Combine with the (all-gathered) vote bitmap through hs_qc_and_dev.
int hs_verify_qc_votes_dev(hs_ctx *c, const void *d_qc_digests, const void *d_pk, const void *d_vidx, const void *d_sig, const void *d_qc_idx,
                           size_t n_votes, void *d_vote_bitmap, void *stream) {
  if (!c || (n_votes && (!d_qc_digests || (!d_pk && !d_vidx) || !d_sig || !d_qc_idx || !d_vote_bitmap)))
    return fail(c, HS_ERR_ARG, "hs_verify_qc_votes_dev: bad argument");
  HS_CUDA(c, cudaSetDevice(c->device));
  in_layout L{(const uint8_t *)d_sig, 64, (const uint8_t *)d_pk, 32, (const uint32_t *)d_vidx, (const uint8_t *)d_qc_digests, 32,
              (const uint32_t *)d_qc_idx, nullptr, 32, 0};
  return run_verify(c, L, n_votes, HS_MODE_BATCH_EQ, (uint32_t *)d_vote_bitmap, (cudaStream_t)stream, d_pk == nullptr);
}
// d_qc_bitmap bit j = AND of the verdict bits of the votes with qc_idx == j (no votes -> 1), over a vote bitmap of n_votes bits.
int hs_qc_and_dev(hs_ctx *c, const void *d_vote_bitmap, const void *d_qc_idx, size_t n_votes, size_t n_qc, void *d_qc_bitmap, void *stream) {
  if (!c || !d_qc_bitmap || (n_votes && (!d_vote_bitmap || !d_qc_idx))) return fail(c, HS_ERR_ARG, "hs_qc_and_dev: bad argument");
  HS_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t st = (c->deferred && (cudaStream_t)stream != c->stream) ? c->stream_tail : (cudaStream_t)stream;  // deferred: after the finish kernel on the tail stream
  if (n_qc) k_bitmap_ones<<<blocks_for((n_qc + 31) / 32, 256), 256, 0, st>>>((uint32_t *)d_qc_bitmap, n_qc);
  c->launches += n_qc ? 1 : 0;
  HS_CUDA(c, cudaGetLastError());
  if (n_votes) HS_TRY(launch_qc_and(c, (const uint32_t *)d_vote_bitmap, (const uint32_t *)d_qc_idx, n_votes, n_qc, (uint32_t *)d_qc_bitmap, st));
  return HS_OK;
}

// ---- device-resident mixed groups: hs_verify_groups with every array in HBM, enqueued on `stream`.  Digest of every preimage
// (k_digest32), then one verify pass whose finish kernel judges item i by d_mode[i], so the item words it writes — locally or into
// every peer's buffer when armed — are final; group verdicts come from hs_qc_and_dev over them.
int hs_verify_groups_dev(hs_ctx *c, const void *d_pre, const void *d_off, size_t n_msgs, const void *d_sig, const void *d_pk, const void *d_vidx,
                         const void *d_msg_idx, const void *d_mode, size_t n_items, void *d_item_bitmap, void *stream) {
  if (!c || (n_items && (!d_pre || !d_off || !d_sig || (!d_pk && !d_vidx) || !d_msg_idx || !d_item_bitmap)))
    return fail(c, HS_ERR_ARG, "hs_verify_groups_dev: bad argument");
  if (n_items && n_msgs == 0) return fail(c, HS_ERR_ARG, "hs_verify_groups_dev: items without preimages");
  if (n_items && !d_pk && !committee_registered(c))
    return fail(c, HS_ERR_ARG, "hs_verify_groups_dev: committee-indexed items without a registered committee");
  HS_CUDA(c, cudaSetDevice(c->device));
  if (n_items == 0) return run_verify(c, in_layout{}, 0, HS_MODE_STRICT, nullptr, (cudaStream_t)stream, false);  // an armed route still signals
  HS_TRY(ensure(c, c->group_digests, n_msgs * 32));
  uint8_t *dig = (uint8_t *)c->group_digests.p.get();
  HS_TRY(hs_digest32_dev(c, d_pre, d_off, n_msgs, dig, stream));
  in_layout L{(const uint8_t *)d_sig, 64, (const uint8_t *)d_pk, 32, (const uint32_t *)d_vidx, dig, 32, (const uint32_t *)d_msg_idx, nullptr, 32, 0};
  return run_verify(c, L, n_items, HS_MODE_STRICT, (uint32_t *)d_item_bitmap, (cudaStream_t)stream, d_pk == nullptr, (const uint8_t *)d_mode);
}

// ---- explanation of a device-resident pass's rejected items (hs_explain_groups_dev): the selection kernels, then k_explain_items on at
// most a quarter of the SMs (the explain lane's share, HS_QUEUE_EXPLAIN_SM_DIV), all on `stream` over scratch of its own.  It records no
// ev_dev_pass: the host-pointer calls do not share its scratch, so they never wait for it.
int hs_explain_groups_dev(hs_ctx *c, const void *d_pre, const void *d_off, size_t n_msgs, const void *d_sig, const void *d_pk, const void *d_msg_idx,
                          const void *d_mode, const void *d_item_bitmap, size_t n_items, size_t max_explain, void *d_why, void *d_out, void *stream) {
  if (!c || (n_items && (!d_pre || !d_off || !d_sig || !d_pk || !d_msg_idx || !d_item_bitmap || !d_why || !d_out)))
    return fail(c, HS_ERR_ARG, "hs_explain_groups_dev: bad argument");
  if (n_items && n_msgs == 0) return fail(c, HS_ERR_ARG, "hs_explain_groups_dev: items without preimages");
  if (n_items > 0xffffffffu) return fail(c, HS_ERR_ARG, "hs_explain_groups_dev: more than 2^32 - 1 items");
  if (n_items == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  const cudaStream_t s = (cudaStream_t)stream;
  const size_t n_words = (n_items + 31) / 32, n_blocks = (n_words + HS_SEL_WORDS - 1) / HS_SEL_WORDS;
  const size_t cap = max_explain && max_explain < n_items ? max_explain : n_items;
  HS_TRY(ensure(c, c->explain_sel, (n_blocks + cap) * 4));
  uint32_t *boff = (uint32_t *)c->explain_sel.p.get(), *list = boff + n_blocks, *out = (uint32_t *)d_out;
  const uint32_t *bm = (const uint32_t *)d_item_bitmap;
  if (c->deferred) HS_TRY(hs_results_wait(c, stream));  // the item words of deferred passes are written on the tail stream
  HS_CUDA(c, cudaMemsetAsync(d_why, HS_WHY_NOT_EXAMINED, n_items, s));
  k_sel_count<<<(unsigned)n_blocks, HS_SEL_WORDS, 0, s>>>(bm, n_items, boff);
  k_sel_top<<<1, HS_SEL_TOP, 0, s>>>(boff, (uint32_t)n_blocks, cap, out);
  k_sel_scatter<<<(unsigned)n_blocks, HS_SEL_WORDS, 0, s>>>(bm, n_items, boff, out, list);
  const unsigned grid = (unsigned)std::min<size_t>(blocks_for(cap), std::max<size_t>(1, c->n_sms / HS_QUEUE_EXPLAIN_SM_DIV));
  k_explain_items<<<grid, HS_THREADS, 0, s>>>(list, (const uint8_t *)d_pre, (const uint64_t *)d_off, (const uint8_t *)d_sig, (const uint8_t *)d_pk,
                                              (const uint32_t *)d_msg_idx, (const uint8_t *)d_mode, (uint8_t *)d_why, out);
  c->launches += 4;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}

// ---- TC::verify / Timeout::verify for many certificates (consensus/src/messages.rs:250-265,290-315)
// Vote i = (key_i, sig_i, high_qc_round_i) of certificate tc_idx[i] (NULL: vote i is its own certificate — the Timeout
// shape, rounds[i] = Timeout.round); message = SHA-512(tc_round || high_qc_round)[..32] built on the GPU; Signature::verify
// (strict) per vote; out_tc_bitmap bit j = AND over certificate j.  Stake / duplicate checks (messages.rs:292-304) stay on the host.
int hs_verify_tcs(hs_ctx *c, const uint64_t *tc_rounds, size_t n_tc, const uint8_t *pk, const uint32_t *vidx, const uint8_t *sig,
                  const uint64_t *high_qc_rounds, const uint32_t *tc_idx, size_t n_votes, uint32_t *out_vote_bitmap, uint32_t *out_tc_bitmap) {
  if (!c || !out_tc_bitmap || (n_tc && !tc_rounds) || (n_votes && (!sig || !high_qc_rounds || (!pk && !vidx) || n_tc == 0)) || (!tc_idx && n_votes && n_tc != n_votes))
    return fail(c, HS_ERR_ARG, "hs_verify_tcs: bad argument");
  if (tc_idx)
    for (size_t i = 0; i < n_votes; i++)
      if (tc_idx[i] >= n_tc) return fail(c, HS_ERR_ARG, "hs_verify_tcs: tc_idx out of range");
  const size_t tc_words = (n_tc + 31) / 32, vote_words = (n_votes + 31) / 32;
  const std::vector<uint32_t> ones = bitmap_ones(n_tc);
  if (n_votes == 0) {
    std::copy(ones.begin(), ones.end(), out_tc_bitmap);
    return HS_OK;
  }
  std::lock_guard<std::mutex> g(c->mu);
  share_call sh(c);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_r = S.add(tc_rounds, n_tc * 8), s_hq = S.add(high_qc_rounds, n_votes * 8), s_dig = S.add(nullptr, n_votes * 32),
               s_sig = S.add(sig, n_votes * 64), s_key = S.add(pk ? (const void *)pk : (const void *)vidx, n_votes * (pk ? 32 : 4)),
               s_ti = S.add(tc_idx, n_votes * 4);
  HS_TRY(ensure(c, c->out, (vote_words + tc_words) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  uint32_t *d_votes = (uint32_t *)c->out.p.get(), *d_tc = d_votes + vote_words;
  const uint32_t *d_ti = tc_idx ? (const uint32_t *)S.ptr(s_ti) : nullptr;
  if (tc_idx) HS_CUDA(c, cudaMemcpyAsync(d_tc, ones.data(), tc_words * 4, cudaMemcpyHostToDevice, c->stream));
  k_tc_digests<<<blocks_for(n_votes), HS_THREADS, 0, c->stream>>>((const uint64_t *)S.ptr(s_r), d_ti, (const uint64_t *)S.ptr(s_hq), n_votes, n_tc,
                                                                  (uint32_t *)S.ptr(s_dig));
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  in_layout L{S.ptr(s_sig), 64, pk ? S.ptr(s_key) : nullptr, 32, pk ? nullptr : (const uint32_t *)S.ptr(s_key), S.ptr(s_dig), 32, nullptr, nullptr, 32, 0};
  HS_TRY(run_verify(c, L, n_votes, HS_MODE_STRICT, d_votes, c->stream, pk == nullptr));
  if (tc_idx) HS_TRY(launch_qc_and(c, d_votes, d_ti, n_votes, n_tc, d_tc, c->stream));
  // without tc_idx, vote i is certificate i
  return readback(c, {{out_vote_bitmap, d_votes, vote_words * 4}, {out_tc_bitmap, tc_idx ? d_tc : d_votes, tc_words * 4}});
}

// ---- mixed groups: Block::verify for many blocks (messages.rs:54-76) = author signature (strict) + QC votes (batch-eq) + TC
// votes (strict), all in ONE pass.  Item i signs Digest(preimage[msg_idx[i]]) (variable-length preimages, hashed on the GPU),
// belongs to group group_idx[i] and is judged by mode[i]; out_group_bitmap bit j = AND over group j's items.
int hs_verify_groups(hs_ctx *c, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                     const uint32_t *vidx, const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *mode, size_t n_items, size_t n_groups,
                     uint32_t *out_item_bitmap, uint32_t *out_group_bitmap) {
  if (!c) return HS_ERR_ARG;
  if (const char *why = hs_args::groups(preimages, pre_off, n_msgs, sig, pk, vidx, msg_idx, group_idx, mode, n_items, n_groups, out_group_bitmap))
    return fail_args(c, "hs_verify_groups", why);
  const size_t g_words = (n_groups + 31) / 32, i_words = (n_items + 31) / 32;
  const std::vector<uint32_t> ones = bitmap_ones(n_groups);
  if (n_items == 0) {
    std::copy(ones.begin(), ones.end(), out_group_bitmap);
    return HS_OK;
  }
  std::lock_guard<std::mutex> g(c->mu);
  share_call sh(c);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_off = S.add(pre_off, (n_msgs + 1) * 8), s_pre = S.add(preimages, pre_off[n_msgs], 8), s_sig = S.add(sig, n_items * 64),
               s_key = S.add(pk ? (const void *)pk : (const void *)vidx, n_items * (pk ? 32 : 4)), s_mi = S.add(msg_idx, n_items * 4),
               s_gi = S.add(group_idx, n_items * 4), s_mo = S.add(mode, n_items);
  HS_TRY(ensure(c, c->out, (i_words + g_words) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  uint32_t *d_items = (uint32_t *)c->out.p.get(), *d_groups = d_items + i_words;
  HS_CUDA(c, cudaMemcpyAsync(d_groups, ones.data(), g_words * 4, cudaMemcpyHostToDevice, c->stream));
  HS_TRY(hs_verify_groups_dev(c, S.ptr(s_pre), S.ptr(s_off), n_msgs, S.ptr(s_sig), pk ? S.ptr(s_key) : nullptr, pk ? nullptr : S.ptr(s_key),
                              S.ptr(s_mi), mode ? S.ptr(s_mo) : nullptr, n_items, d_items, c->stream));
  HS_TRY(launch_qc_and(c, d_items, (const uint32_t *)S.ptr(s_gi), n_items, n_groups, d_groups, c->stream));
  return readback(c, {{out_item_bitmap, d_items, i_words * 4}, {out_group_bitmap, d_groups, g_words * 4}});
}

// ---- load generation (SURVEY §8f.4): RFC 8032 keygen / signing of 32-byte digests on the GPU
int hs_keygen_batch_dev(hs_ctx *c, const void *d_seeds, size_t n, void *d_pks, void *stream) {
  if (!c || (n && (!d_seeds || !d_pks))) return fail(c, HS_ERR_ARG, "hs_keygen_batch_dev: bad argument");
  if (n == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  k_keygen<<<blocks_for(n), HS_THREADS, 0, (cudaStream_t)stream>>>((const uint8_t *)d_seeds, n, c->d_btable, c->cp, (uint8_t *)d_pks);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
int hs_sign_digests_dev(hs_ctx *c, const void *d_seeds, const void *d_pks, size_t n_keys, const void *d_key_idx, const void *d_digests, size_t n,
                        void *d_sig, void *stream) {
  if (!c || (n && (!d_seeds || !d_pks || !d_digests || !d_sig || n_keys == 0)) || (!d_key_idx && n > n_keys))
    return fail(c, HS_ERR_ARG, "hs_sign_digests_dev: bad argument");
  if (n == 0) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  k_sign_digests<<<blocks_for(n), HS_THREADS, 0, (cudaStream_t)stream>>>((const uint8_t *)d_seeds, (const uint8_t *)d_pks, (const uint32_t *)d_key_idx,
                                                                          (const uint8_t *)d_digests, n, n_keys, c->d_btable, c->cp, (uint8_t *)d_sig);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}
int hs_keygen_batch(hs_ctx *c, const uint8_t *seeds, size_t n, uint8_t *out_pks) {
  if (!c || (n && (!seeds || !out_pks))) return fail(c, HS_ERR_ARG, "hs_keygen_batch: bad argument");
  if (n == 0) return HS_OK;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_seed = S.add(seeds, n * 32);
  HS_TRY(ensure(c, c->out, n * 32));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  HS_TRY(hs_keygen_batch_dev(c, S.ptr(s_seed), n, c->out.p, c->stream));
  return readback(c, {{out_pks, c->out.p.get(), n * 32}});
}
int hs_sign_digests(hs_ctx *c, const uint8_t *seeds, const uint8_t *pks, size_t n_keys, const uint32_t *key_idx, const uint8_t *digests, size_t n,
                    uint8_t *out_sig) {
  if (!c || (n && (!seeds || !pks || !digests || !out_sig || n_keys == 0)) || (!key_idx && n > n_keys)) return fail(c, HS_ERR_ARG, "hs_sign_digests: bad argument");
  if (n == 0) return HS_OK;
  if (key_idx)
    for (size_t i = 0; i < n; i++)
      if (key_idx[i] >= n_keys) return fail(c, HS_ERR_ARG, "hs_sign_digests: key index out of range");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_seed = S.add(seeds, n_keys * 32), s_pk = S.add(pks, n_keys * 32), s_ki = S.add(key_idx, n * 4), s_d = S.add(digests, n * 32);
  HS_TRY(ensure(c, c->out, n * 64));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  HS_TRY(hs_sign_digests_dev(c, S.ptr(s_seed), S.ptr(s_pk), n_keys, key_idx ? S.ptr(s_ki) : nullptr, S.ptr(s_d), n, c->out.p, c->stream));
  return readback(c, {{out_sig, c->out.p.get(), n * 64}});
}

// ---- multi-GPU peer routing (one process per GPU; handles are exchanged by the host, e.g. torch.distributed.all_gather_object)
int hs_peer_setup(hs_ctx *c, int rank, int world, size_t total_words, uint8_t handle_out[64]) {
  if (!c || world < 1 || world > HS_MAX_PEERS || rank < 0 || rank >= world || !handle_out || total_words % (size_t)world)
    return fail(c, HS_ERR_ARG, "hs_peer_setup: bad argument (total_words must be a multiple of world)");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  if (c->peer.own) {  // a new geometry (another workload): drop the old buffers.  Every rank must have drained its stream first.
    HS_CUDA(c, cudaDeviceSynchronize());
    c->peer = {};  // nothing points at them after this: a failure below leaves peer routing unset
    c->peers = peer_route{};
    c->peer_epoch = 0;
    c->peer_armed = false;
  }
  const size_t bytes = (2 * total_words + HS_MAX_PEERS + 16) * 4;
  dev_mem<uint32_t> own;
  HS_CUDA(c, alloc(own, bytes));
  HS_CUDA(c, cudaMemset(own, 0, bytes));
  cudaIpcMemHandle_t h;
  HS_CUDA(c, cudaIpcGetMemHandle(&h, own));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, 64);
  c->peer.own = std::move(own);
  c->peer_rank = rank;
  c->peer_total_words = total_words;
  c->peers = peer_route{};
  c->peers.n = world;
  c->peers.my_rank = rank;
  c->peers.total_words = total_words;
  c->peers.buf[rank] = c->peer.own;
  return HS_OK;
}
int hs_peer_open(hs_ctx *c, int peer_rank, const uint8_t handle[64]) {
  if (!c || !handle || peer_rank < 0 || peer_rank >= c->peers.n || peer_rank == c->peer_rank) return fail(c, HS_ERR_ARG, "hs_peer_open: bad argument");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  ipc_mapping &m = c->peer.mapped[peer_rank];
  if (m) HS_CUDA(c, cudaDeviceSynchronize());  // reopened: a pass may still write through the earlier mapping, closed below
  c->peers.buf[peer_rank] = nullptr;
  HS_CUDA(c, ipc_open(m, h));
  c->peers.buf[peer_rank] = static_cast<uint32_t *>(m.get());
  return HS_OK;
}
/* Arms the NEXT `_dev` verify call on this context: its bitmap goes to every rank's buffer at word_offset (fused all-gather). */
int hs_peer_next(hs_ctx *c, size_t word_offset, uint32_t epoch) {
  if (!c || !c->peer.own) return fail(c, HS_ERR_ARG, "hs_peer_next: peers not set up");
  std::lock_guard<std::mutex> g(c->mu);
  for (int p = 0; p < c->peers.n; p++)
    if (!c->peers.buf[p]) return fail(c, HS_ERR_ARG, "hs_peer_next: a peer buffer is not mapped");
  if (c->peer_epoch != 0 && epoch != c->peer_epoch + 1) return fail(c, HS_ERR_ARG, "hs_peer_next: epochs must increase by one");
  if (word_offset >= c->peer_total_words && c->peer_total_words) return fail(c, HS_ERR_ARG, "hs_peer_next: word_offset out of range");
  c->peers.word_offset = word_offset;
  c->peers.epoch = epoch;
  c->peer_epoch = epoch;
  c->peer_armed = true;
  return HS_OK;
}
/* Device pointer of this rank's copy of the full bitmap of the most recently armed epoch, and whether a peer wait ever timed out. */
void *hs_peer_bitmap(hs_ctx *c) { return (c && c->peer.own) ? (void *)(c->peer.own + (size_t)(c->peer_epoch & 1u) * c->peer_total_words) : nullptr; }
int hs_peer_timed_out(hs_ctx *c) {
  if (!c || !c->peer.own) return 0;
  uint32_t v = 0;
  cudaSetDevice(c->device);
  cudaMemcpy(&v, c->peer.own + 2 * c->peer_total_words + HS_MAX_PEERS, 4, cudaMemcpyDeviceToHost);
  return (int)v;
}

// ---- host-pointer entry points
int hs_verify_rec128(hs_ctx *c, const hs_rec128 *recs, size_t n, uint32_t mode, uint32_t *out_bitmap) {
  if (!c) return HS_ERR_ARG;
  if (const char *why = hs_args::rec128(recs, n, mode, out_bitmap)) return fail_args(c, "hs_verify_rec128", why);
  if (n == 0) return HS_OK;
  std::lock_guard<std::mutex> g(c->mu);
  share_call sh(c);
  HS_CUDA(c, cudaSetDevice(c->device));
  // latency path: every key must already have a table (registered or learned)
  if (small_eligible(c, n) && small_stage(c, n, [&](size_t i) { return small_src{recs[i].sig, recs[i].msg, host_key_lookup(c, recs[i].pk)}; }))
    return run_small(c, n, mode, out_bitmap);
  h2d_stage S;
  const size_t s_recs = S.add(recs, n * sizeof(hs_rec128));
  HS_TRY(ensure(c, c->out, ((n + 31) / 32) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  HS_TRY(hs_verify_rec128_dev(c, S.ptr(s_recs), n, mode, c->out.p, c->stream));
  return readback(c, {{out_bitmap, c->out.p.get(), ((n + 31) / 32) * 4}});
}
int hs_verify_strict_batch(hs_ctx *c, const hs_rec128 *recs, size_t n, uint32_t *out_bitmap) {
  return hs_verify_rec128(c, recs, n, HS_MODE_STRICT, out_bitmap);
}

int hs_verify_var(hs_ctx *c, const uint8_t *sig, const uint8_t *pk, const uint8_t *msgs, const uint64_t *off, size_t n, uint32_t mode,
                  uint32_t *out_bitmap) {
  if (!c || mode > 1 || (n && (!sig || !pk || !off || !out_bitmap))) return fail(c, HS_ERR_ARG, "hs_verify_var: bad argument");
  if (n == 0) return HS_OK;
  if (!offsets_ok(off, n)) return fail(c, HS_ERR_ARG, "hs_verify_var: offsets must start at 0 and be non-decreasing");
  if (off[n] && !msgs) return fail(c, HS_ERR_ARG, "hs_verify_var: null msgs");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_sig = S.add(sig, n * 64), s_pk = S.add(pk, n * 32), s_off = S.add(off, (n + 1) * 8), s_msg = S.add(msgs, off[n], 8);
  HS_TRY(ensure(c, c->out, ((n + 31) / 32) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  HS_TRY(hs_verify_var_dev(c, S.ptr(s_sig), S.ptr(s_pk), S.ptr(s_msg), S.ptr(s_off), n, mode, c->out.p, c->stream));
  return readback(c, {{out_bitmap, c->out.p.get(), ((n + 31) / 32) * 4}});
}

int hs_verify_batch_shared_msg(hs_ctx *c, const uint8_t digest[32], const hs_vote *votes, size_t n, int *all_ok, uint32_t *out_bitmap_or_null) {
  if (!c || !all_ok || !digest || (n && !votes)) return fail(c, HS_ERR_ARG, "hs_verify_batch_shared_msg: bad argument");
  *all_ok = 0;
  if (n == 0) {  // dalek::verify_batch on empty input is Ok
    *all_ok = 1;
    return HS_OK;
  }
  std::lock_guard<std::mutex> g(c->mu);
  share_call sh(c);
  HS_CUDA(c, cudaSetDevice(c->device));
  const size_t words = (n + 31) / 32;
  std::vector<uint32_t> tmp;
  uint32_t *bm = out_bitmap_or_null;
  if (!bm) {
    tmp.resize(words);
    bm = tmp.data();
  }
  // latency path (the 2f+1 = 3 votes of a 4-node QC)
  if (small_eligible(c, n) && small_stage(c, n, [&](size_t i) { return small_src{votes[i].sig, digest, host_key_lookup(c, votes[i].pk)}; })) {
    HS_TRY(run_small(c, n, HS_MODE_BATCH_EQ, bm));
  } else {
    h2d_stage S;
    const size_t s_dig = S.add(digest, 32), s_votes = S.add(votes, n * sizeof(hs_vote));
    HS_TRY(ensure(c, c->out, words * 4));
    HS_TRY(S.upload(c, c->in[0], c->stream));
    const uint8_t *v = S.ptr(s_votes);  // hs_vote: pk | sig
    in_layout L{v + 32, sizeof(hs_vote), v, sizeof(hs_vote), nullptr, S.ptr(s_dig), 0, nullptr, nullptr, 32, 0};
    HS_TRY(run_verify(c, L, n, HS_MODE_BATCH_EQ, (uint32_t *)c->out.p.get(), c->stream, false));
    HS_TRY(readback(c, {{bm, c->out.p.get(), words * 4}}));
  }
  int ok = 1;
  for (size_t w = 0; w < words; w++)
    if (bm[w] != bitmap_word_ones(n, w)) ok = 0;
  *all_ok = ok;
  return HS_OK;
}

int hs_verify_committee(hs_ctx *c, const uint32_t *vidx, const uint8_t *sig, const uint32_t *midx, const uint8_t *digests, size_t n_msgs,
                        size_t n, uint32_t mode, uint32_t *out_bitmap) {
  if (!c || mode > 1 || (n && (!vidx || !sig || !digests || !out_bitmap || n_msgs == 0)) || (n && !midx && n_msgs != 1))
    return fail(c, HS_ERR_ARG, "hs_verify_committee: bad argument");
  if (n == 0) return HS_OK;
  if (midx)
    for (size_t i = 0; i < n; i++)
      if (midx[i] >= n_msgs) return fail(c, HS_ERR_ARG, "hs_verify_committee: msg_idx out of range");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  if (small_eligible(c, n) && committee_registered(c)) {  // latency path: the indices as given (the kernel rejects one without a key)
    small_stage(c, n, [&](size_t i) { return small_src{sig + 64 * i, digests + 32 * (size_t)(midx ? midx[i] : 0), vidx[i]}; });
    return run_small(c, n, mode, out_bitmap);
  }
  h2d_stage S;
  const size_t s_sig = S.add(sig, n * 64), s_v = S.add(vidx, n * 4), s_m = S.add(midx, midx ? n * 4 : 0), s_d = S.add(digests, n_msgs * 32);
  HS_TRY(ensure(c, c->out, ((n + 31) / 32) * 4));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  HS_TRY(hs_verify_committee_dev(c, S.ptr(s_v), S.ptr(s_sig), midx ? S.ptr(s_m) : nullptr, S.ptr(s_d), n, mode, c->out.p, c->stream));
  return readback(c, {{out_bitmap, c->out.p.get(), ((n + 31) / 32) * 4}});
}

int hs_digest32_batch(hs_ctx *c, const uint8_t *data, const uint64_t *off, size_t n, uint8_t *out) {
  if (!c || (n && (!off || !out))) return fail(c, HS_ERR_ARG, "hs_digest32_batch: bad argument");
  if (n == 0) return HS_OK;
  if (!offsets_ok(off, n)) return fail(c, HS_ERR_ARG, "hs_digest32_batch: offsets must start at 0 and be non-decreasing");
  if (off[n] && !data) return fail(c, HS_ERR_ARG, "hs_digest32_batch: null data");
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_off = S.add(off, (n + 1) * 8), s_data = S.add(data, off[n], 8);
  HS_TRY(ensure(c, c->out, n * 32));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  if (n <= 64 && off[n] / n >= 1024)  // a few long messages (mempool batches)
    HS_TRY(launch_digest_long(c, S.ptr(s_data), (const uint64_t *)S.ptr(s_off), n, (uint32_t *)c->out.p.get(), c->stream));
  else
    HS_TRY(hs_digest32_dev(c, S.ptr(s_data), S.ptr(s_off), n, c->out.p, c->stream));
  return readback(c, {{out, c->out.p.get(), n * 32}});
}

// Reference-shaped end-to-end call: verdict_i = Signature::verify(Digest(msg_i), key_i) for fixed-size messages, with the
// H2D copy of chunk j+1 overlapped with the kernels of chunk j (two streams, two staging buffers).
int hs_verify_msgs(hs_ctx *c, const uint8_t *sig, const uint8_t *pk, const uint32_t *vidx, const uint8_t *msgs, size_t msg_len, size_t n,
                   uint32_t mode, uint32_t *out_bitmap) {
  if (!c) return HS_ERR_ARG;
  if (const char *why = hs_args::msgs(sig, pk, vidx, msgs, msg_len, n, mode, out_bitmap)) return fail_args(c, "hs_verify_msgs", why);
  if (n == 0) return HS_OK;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  size_t CH = 1u << 17;  // records per chunk (multiple of 32): every chunk with an unknown key waits for the single-warp latency of the
                         // generic pass, so chunks must be long enough for the PCIe copy of the next chunk to cover it
  if (const char *e = getenv("HS_CHUNK_RECORDS")) {
    size_t v = strtoull(e, nullptr, 10);
    if (v >= 1024) CH = v & ~(size_t)31;
  }
  const size_t key_bytes = vidx ? 4 : 32;
  const size_t per_rec = 64 + key_bytes + msg_len;
  const size_t chunk_cap = (n < CH ? n : CH);
  HS_TRY(ensure(c, c->out, ((n + 31) / 32) * 4));
  // scratch shared by both chunks' verify passes is stream-ordered: verify of chunk j+1 is enqueued on the same compute
  // stream after chunk j, only the copies run ahead on the second stream.
  for (int b = 0; b < 2; b++) {
    HS_TRY(ensure(c, c->in[b], chunk_cap * per_rec + 64));
    HS_TRY(ensure(c, c->digest[b], chunk_cap * 32));
  }
  HS_TRY(ensure(c, c->xyz, chunk_cap * 3 * sizeof(fe)));
  HS_TRY(ensure(c, c->meta, chunk_cap));
  if (!vidx && has_key_tables(c)) {
    HS_TRY(ensure(c, c->vidx, chunk_cap * 4));
    HS_TRY(ensure(c, c->miss, chunk_cap * 4));
  }
  // (A short "ramp" first chunk was tried and measured slower — 7.1e7 vs 7.6e7 verifies/s: every extra chunk costs one more
  // generic-pass latency when the batch contains unknown keys.)
  // The chunks' passes reuse the verify scratch on `stream`, after any `_dev` pass that may still read it (staging on stream2 does not)
  HS_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_dev_pass, 0));
  size_t lo = 0;
  for (size_t j = 0; lo < n; j++) {
    const int b = (int)(j & 1);
    const size_t cnt = (n - lo < CH) ? (n - lo) : CH;
    uint8_t *d = (uint8_t *)c->in[b].p.get();
    const size_t o_sig = 0, o_key = cnt * 64, o_msg = o_key + ((cnt * key_bytes + 15) & ~(size_t)15);
    if (j >= 2) HS_CUDA(c, cudaStreamWaitEvent(c->stream2, c->ev_done[b], 0));  // staging buffer b is free again
    HS_CUDA(c, cudaMemcpyAsync(d + o_sig, sig + lo * 64, cnt * 64, cudaMemcpyHostToDevice, c->stream2));
    if (vidx) HS_CUDA(c, cudaMemcpyAsync(d + o_key, vidx + lo, cnt * 4, cudaMemcpyHostToDevice, c->stream2));
    else HS_CUDA(c, cudaMemcpyAsync(d + o_key, pk + lo * 32, cnt * 32, cudaMemcpyHostToDevice, c->stream2));
    HS_CUDA(c, cudaMemcpyAsync(d + o_msg, msgs + lo * msg_len, cnt * msg_len, cudaMemcpyHostToDevice, c->stream2));
    HS_CUDA(c, cudaEventRecord(c->ev[b], c->stream2));
    HS_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev[b], 0));
    HS_TRY(hs_verify_msgs_dev(c, d + o_sig, vidx ? nullptr : d + o_key, vidx ? d + o_key : nullptr, d + o_msg, msg_len, cnt, mode,
                              c->digest[b].p, (uint32_t *)c->out.p.get() + lo / 32, c->stream));
    HS_CUDA(c, cudaEventRecord(c->ev_done[b], c->stream));
    lo += cnt;
  }
  return readback(c, {{out_bitmap, c->out.p.get(), ((n + 31) / 32) * 4}});
}

// ---- verify queue
int hs_queue_create(hs_ctx *c, size_t ring_records, hs_queue **out) {
  if (!c || !out || ring_records > HS_QUEUE_MAX_RECORDS) return fail(c, HS_ERR_ARG, "hs_queue_create: bad argument");
  *out = nullptr;
  uint32_t cap = HS_SMALL_MAX;  // a request of 64 records must fit
  while (cap < (ring_records ? ring_records : HS_QUEUE_DEFAULT_RECORDS)) cap <<= 1;
  HS_CUDA(c, cudaSetDevice(c->device));
  std::unique_ptr<hs_queue> q(new (std::nothrow) hs_queue());  // on failure below, its owners release what was allocated
  if (!q) return fail(c, HS_ERR_NOMEM, "hs_queue_create: out of host memory");
  q->c = c;
  q->cap = cap;
  q->mask = cap - 1;
  q->arena.cap = cap * HS_QUEUE_ARENA_PER_RECORD;
  q->modes.assign(cap, 0);
  q->wbits.assign(cap / 32, 0);
  q->reqs.assign(cap, hs_queue::req{});
  int lo = 0, hi = 0;
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (e == cudaSuccess) e = create(q->stream, hi);
  if (e == cudaSuccess) e = create(q->bulk_stream, lo);
  if (e == cudaSuccess) e = create(q->ev_last);
  if (e == cudaSuccess) e = create(q->ev_bulk_last);
  if (e == cudaSuccess) e = make_ring(q->ring, cap, q->stream);
  if (e == cudaSuccess) e = alloc(q->arena_buf, q->arena.cap);
  if (e == cudaSuccess) e = alloc(q->mlist, (size_t)cap * sizeof(qmsg_desc));
  if (e == cudaSuccess) e = alloc(q->pk, (size_t)cap * 32);
  if (e == cudaSuccess) e = alloc(q->d_stage, q->arena.cap);
  if (e == cudaSuccess) e = alloc(q->d_digs, q->arena.cap * 4);
  if (e != cudaSuccess) return fail(c, HS_ERR_CUDA, "hs_queue_create", e);
  memset(q->pk.h, 0, (size_t)cap * 32);
  try {
    q->th = std::thread(queue_main, q.get());
  } catch (...) {
    return fail(c, HS_ERR_NOMEM, "hs_queue_create: cannot start the dispatcher thread");
  }
  {
    std::lock_guard<std::mutex> g(c->queues_mu);
    c->queues.push_back(q.get());
  }
  *out = q.release();
  return HS_OK;
}

// The records of one request that enter the ring: record sel[k] of the caller's arrays (k itself when sel is null), k < n.
struct queue_sel {
  const uint32_t *sel;
  size_t n;
  size_t operator[](size_t k) const { return sel ? sel[k] : k; }
};

// Copies one request's selected records into the ring (under q->mu, arguments already checked) as ring request r: record i is
// judged by modes[i], or by `mode` when modes is null.  HS_ERR_NOMEM when the ring has no room.
static int queue_put_recs_locked(hs_queue *q, const char *what, const hs_rec128 *recs, queue_sel sel, uint32_t mode, const uint8_t *modes,
                                 hs_queue::req r) {
  if (sel.n > q->cap) return fail(q->c, HS_ERR_ARG, (std::string(what) + ": more records than the ring holds").c_str());
  if (q->tail - q->head + sel.n > q->cap) return HS_ERR_NOMEM;  // ring full: back-pressure, not an engine failure
  for (size_t k = 0; k < sel.n; k++) {
    const size_t i = sel[k];
    const uint32_t s = (uint32_t)((q->tail + k) & q->mask);
    memcpy(q->ring.recs.h[s].sig, recs[i].sig, 64);
    memcpy(q->ring.recs.h[s].msg, recs[i].msg, 32);
    memcpy(q->pk.h + 32 * (size_t)s, recs[i].pk, 32);
    q->modes[s] = modes ? modes[i] : (uint8_t)mode;
  }
  r.n = (uint32_t)sel.n;
  q->reqs[q->tail & q->mask] = r;
  q->tail += sel.n;
  return HS_OK;
}

// The same for a preimage request: the selected records go into the ring and the preimages they name, in their order, into one
// arena region.  HS_ERR_ARG when the region is larger than the arena, HS_ERR_NOMEM when the arena or the ring has no room.
static int queue_put_msgs_locked(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                                 const uint32_t *msg_idx, const uint8_t *modes, queue_sel sel, hs_queue::req r) {
  const size_t n = sel.n;
  if (n > q->cap) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_msgs: more records than the ring holds");
  // keep only the preimages some record names, in their order: remap[j] = new index of preimage j
  std::vector<uint32_t> remap(n_msgs, HS_NO_KEY);
  for (size_t k = 0; k < n; k++) remap[msg_idx[sel[k]]] = 0;
  uint32_t m = 0;
  uint64_t pre_bytes = 0;
  for (size_t j = 0; j < n_msgs; j++)
    if (remap[j] == 0) {
      remap[j] = m++;
      pre_bytes += pre_off[j + 1] - pre_off[j];
    }
  const uint64_t size = qmsg_bytes(m, n, pre_bytes);
  if (size > q->arena.cap) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_msgs: more preimage bytes than the queue's arena holds");
  const std::optional<uint64_t> start = q->arena.take(size);
  if (!start) return HS_ERR_NOMEM;
  if (q->tail - q->head + n > q->cap) return HS_ERR_NOMEM;  // ring full: back-pressure, not an engine failure
  uint8_t *a = q->arena_buf.h + q->arena.off(*start);
  uint64_t *off = reinterpret_cast<uint64_t *>(a);
  uint32_t *idx = reinterpret_cast<uint32_t *>(a + 8 * ((size_t)m + 1));
  uint8_t *pre = a + qmsg_o_pre(m, n);
  off[0] = 0;
  for (size_t j = 0, k = 0; j < n_msgs; j++)
    if (remap[j] != HS_NO_KEY) {
      const uint64_t len = pre_off[j + 1] - pre_off[j];
      if (len) memcpy(pre + off[k], preimages + pre_off[j], len);
      off[k + 1] = off[k] + len;
      k++;
    }
  for (size_t k = 0; k < n; k++) {
    const size_t i = sel[k];
    const uint32_t s = (uint32_t)((q->tail + k) & q->mask);
    memcpy(q->ring.recs.h[s].sig, sig + 64 * i, 64);
    memcpy(q->pk.h + 32 * (size_t)s, pk + 32 * i, 32);
    q->modes[s] = modes ? modes[i] : (uint8_t)HS_MODE_STRICT;
    idx[k] = remap[msg_idx[i]];
  }
  r.n = (uint32_t)n;
  r.msgs = true;
  r.a_off = (uint32_t)q->arena.off(*start);
  r.m = m;
  r.pre_bytes = (uint32_t)pre_bytes;
  r.a_end = q->arena.tail = *start + size;
  q->reqs[q->tail & q->mask] = r;
  q->tail += n;
  q->dstats[3]++;
  return HS_OK;
}

// A request's spans (see cert_key): record i signs msg(i) with key pk(i) (32 bytes) and signature sig(i) (64 bytes).  Null when
// the request has no span; its records then all enter the ring exactly as with the cache off.
extern "C++" {
template <class Msg, class Pk, class Sig>
static std::unique_ptr<cert_req> cert_spans(char kind, size_t n, const uint8_t *modes, hs_queue_cb *cb, void *user, Msg msg, Pk pk, Sig sig) {
  if (!modes) return nullptr;  // all strict
  std::unordered_map<std::string_view, size_t> by_msg;
  std::vector<std::vector<uint32_t>> groups;
  for (uint32_t i = 0; i < n; i++) {
    if (modes[i] != HS_MODE_BATCH_EQ) continue;
    auto it = by_msg.emplace(msg(i), groups.size()).first;
    if (it->second == groups.size()) groups.emplace_back();
    groups[it->second].push_back(i);
  }
  std::unique_ptr<cert_req> cr;
  for (std::vector<uint32_t> &g : groups) {
    if (g.size() < 2) continue;
    if (!cr) cr.reset(new cert_req{{0, cb, user}, (uint32_t)n, {}, {}, 0, HS_OK, std::vector<uint32_t>((n + 31) / 32, 0u)});
    const std::string_view m = msg(g[0]);
    const uint64_t len = m.size();
    std::string key;
    key.reserve(1 + 8 + m.size() + 96 * g.size());
    key.push_back(kind);
    key.append(reinterpret_cast<const char *>(&len), 8);
    key.append(m);
    for (uint32_t i : g) {
      key.append(reinterpret_cast<const char *>(pk(i)), 32);
      key.append(reinterpret_cast<const char *>(sig(i)), 64);
    }
    const size_t h = std::hash<std::string_view>{}(key);
    cr->spans.push_back(cert_span{std::move(key), h, std::move(g), CERT_NEW});
  }
  return cr;
}

// Submits one request of any kind: under q->mu, put(s) takes the request's room and records it with sink s (s.ticket is the ticket
// it gets), returning HS_OK, or an error that leaves the queue as it was.  The ticket is issued only when put accepted the request.
template <class Put>
static int queue_submit(hs_queue *q, const char *what, ticket_sink s, uint32_t n_bits, size_t *out_ticket, Put put) {
  {
    std::lock_guard<std::mutex> g(q->mu);
    if (q->stop) return fail(q->c, HS_ERR_ARG, (std::string(what) + ": queue is being destroyed").c_str());
    s.ticket = q->next_ticket;
    const int rc = put(s);
    if (rc != HS_OK) return rc;
    ticket_open_locked(q, s, n_bits);
    if (out_ticket) *out_ticket = s.ticket;
  }
  q->cv_work.notify_one();
  return HS_OK;
}

// Submits a request that has spans, with the cache on.  Under q->mu each span is a hit, a join of an identical span pending or in
// flight in an earlier request, or new; `put(sel, r)` enters the records of no hit or joined span into the ring as request r.  When
// there are none the request is answered entirely here and the queue's thread completes it.  Nothing changes on an error.
template <class Put>
static int cert_submit(hs_queue *q, const char *what, std::unique_ptr<cert_req> cr, size_t *out_ticket, Put put) {
  std::vector<int32_t> span_of(cr->n, -1);
  for (size_t j = 0; j < cr->spans.size(); j++)
    for (uint32_t i : cr->spans[j].idx) span_of[i] = (int32_t)j;
  return queue_submit(q, what, cr->sink, cr->n, out_ticket, [&](const ticket_sink &s) {
    for (cert_span &sp : cr->spans) {
      const cert_key k{sp.h, sp.key};
      sp.role = q->cc_map.count(k) ? CERT_HIT : q->cc_flights.count(k) ? CERT_JOINED : CERT_NEW;
    }
    std::vector<uint32_t> sel;
    for (uint32_t i = 0; i < cr->n; i++)
      if (span_of[i] < 0 || cr->spans[span_of[i]].role == CERT_NEW) sel.push_back(i);
    if (!sel.empty()) {
      hs_queue::req r{};
      r.cr = cr.get();
      const int rc = put(queue_sel{sel.data(), sel.size()}, r);
      if (rc != HS_OK) return rc;
      cr->pending++;
    }
    cr->ring_idx = std::move(sel);
    cr->sink = s;
    q->cstats[0] += cr->spans.size();
    for (cert_span &sp : cr->spans) {
      const cert_key k{sp.h, sp.key};
      if (sp.role == CERT_HIT) {
        auto it = q->cc_map.find(k);
        q->cc_lru.splice(q->cc_lru.begin(), q->cc_lru, it->second);
        for (uint32_t i : sp.idx) cr->bits[i >> 5] |= 1u << (i & 31);
        q->cstats[1]++;
      } else if (sp.role == CERT_JOINED) {
        q->cc_flights.find(k)->second.joiners.emplace_back(cr.get(), &sp);
        cr->pending++;
        q->cstats[2]++;
      } else {
        q->cc_flights.emplace(k, cert_flight{});
        continue;
      }
      q->cstats[3] += sp.idx.size();
    }
    if (cr->pending == 0) q->cc_ready.push_back(cr.get());
    cr.release();  // owned by the queue until it completes
    return HS_OK;
  });
}

// Reads one of the queue's counter arrays for an hs_queue_*stats entry point.
template <size_t N>
static int queue_read_stats(hs_queue *q, const char *what, uint64_t *out, uint64_t (hs_queue::*arr)[N]) {
  if (!q || !out) return fail(q ? q->c : nullptr, HS_ERR_ARG, (std::string(what) + ": bad argument").c_str());
  std::lock_guard<std::mutex> g(q->mu);
  q->cstats[5] = q->cc_bytes;  // hs_queue_cert_stats' [5]: the key bytes held now
  memcpy(out, q->*arr, sizeof(q->*arr));
  return HS_OK;
}
// The same for the first n counters of a side lane's.
static int queue_read_stats(hs_queue *q, const char *what, uint64_t *out, side_lane hs_queue::*lane, size_t n) {
  if (!q || !out) return fail(q ? q->c : nullptr, HS_ERR_ARG, (std::string(what) + ": bad argument").c_str());
  std::lock_guard<std::mutex> g(q->mu);
  memcpy(out, (q->*lane).stats, 8 * n);
  return HS_OK;
}

// Submits request r to lane L: under q->mu it checks that the lane is on and that r fits the lane's limits, takes r's region of the
// arena and joins the lane's list; then fill(region) writes its inputs without the lock, its result words and tail are zeroed, and it
// becomes ready.  The region is the request's alone until it completes.
template <class Fill>
static int lane_submit(hs_queue *q, side_lane &L, const char *what, lane_req r, size_t *out_ticket, Fill fill) {
  lane_req *p = nullptr;
  const int rc = queue_submit(q, what, r.sink, r.n_bits, out_ticket, [&](const ticket_sink &s) {
    if (!L.max_recs) return fail(q->c, HS_ERR_ARG, (std::string(what) + ": the " + L.kind.name + " lane is off (" + L.kind.configure + ")").c_str());
    if (r.n > L.max_recs || r.size > L.max_bytes)
      return fail(q->c, HS_ERR_ARG, (std::string(what) + ": larger than the " + L.kind.name + " lane's limits").c_str());
    const std::optional<uint64_t> start = L.ring.take(r.size);
    if (!start) return HS_ERR_NOMEM;
    r.sink = s;
    r.a_off = L.ring.off(*start);
    r.a_pos = *start;
    r.a_end = L.ring.tail = *start + r.size;
    L.reqs.push_back(r);
    p = &L.reqs.back();  // stays valid: only the dispatcher pops, and never a request that is not ready
    return HS_OK;
  });
  if (rc != HS_OK) return rc;
  uint8_t *a = L.buf.arena.h + p->a_off;
  fill(a);
  memset(a + p->o_res, 0, p->size - p->o_res);  // result words and the tail
  {
    std::lock_guard<std::mutex> g(q->mu);
    p->ready = true;
  }
  q->cv_work.notify_one();
  return HS_OK;
}
}  // extern "C++"

int hs_queue_submit(hs_queue *q, const hs_rec128 *recs, size_t n, uint32_t mode, hs_queue_cb *cb, void *user, size_t *out_ticket) {
  if (!q || !recs || n == 0 || n > HS_SMALL_MAX || mode > 1) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit: bad argument");
  return queue_submit(q, "hs_queue_submit", ticket_sink{0, cb, user}, (uint32_t)n, out_ticket, [&](const ticket_sink &s) {
    return queue_put_recs_locked(q, "hs_queue_submit", recs, queue_sel{nullptr, n}, mode, nullptr, hs_queue::req{s});
  });
}

// With the certificate cache on, the ring capacity limits the records that enter the ring (checked under the lock), not n.
#define HS_QUEUE_CERT_MAX_N ((size_t)UINT32_MAX)

int hs_queue_submit_group(hs_queue *q, const hs_rec128 *recs, size_t n, const uint8_t *modes, hs_queue_cb *cb, void *user, size_t *out_ticket) {
  const bool cache = q && q->cc_max.load() > 0;
  if (!q || !recs || n == 0 || n > (cache ? HS_QUEUE_CERT_MAX_N : q->cap)) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit_group: bad argument");
  if (modes)
    for (size_t i = 0; i < n; i++)
      if (modes[i] > HS_MODE_BATCH_EQ) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_group: bad mode byte");
  std::unique_ptr<cert_req> cr;
  if (cache)
    cr = cert_spans('D', n, modes, cb, user, [&](size_t i) { return std::string_view(reinterpret_cast<const char *>(recs[i].msg), 32); },
                    [&](size_t i) { return recs[i].pk; }, [&](size_t i) { return recs[i].sig; });
  const auto put = [&](queue_sel sel, const hs_queue::req &r) {
    return queue_put_recs_locked(q, "hs_queue_submit_group", recs, sel, HS_MODE_STRICT, modes, r);
  };
  if (cr) return cert_submit(q, "hs_queue_submit_group", std::move(cr), out_ticket, put);
  if (n > q->cap) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_group: bad argument");
  return queue_submit(q, "hs_queue_submit_group", ticket_sink{0, cb, user}, (uint32_t)n, out_ticket,
                      [&](const ticket_sink &s) { return put(queue_sel{nullptr, n}, hs_queue::req{s}); });
}

int hs_queue_submit_msgs(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                         const uint32_t *msg_idx, const uint8_t *modes, size_t n, hs_queue_cb *cb, void *user, size_t *out_ticket) {
  const bool cache = q && q->cc_max.load() > 0;
  if (!q || !pre_off || !sig || !pk || !msg_idx || n == 0 || n > (cache ? HS_QUEUE_CERT_MAX_N : q->cap) || n_msgs == 0)
    return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit_msgs: bad argument");
  if (!offsets_ok(pre_off, n_msgs) || (pre_off[n_msgs] && !preimages)) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_msgs: bad preimage offsets");
  for (size_t i = 0; i < n; i++)
    if (msg_idx[i] >= n_msgs || (modes && modes[i] > HS_MODE_BATCH_EQ)) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_msgs: index or mode out of range");
  std::unique_ptr<cert_req> cr;
  if (cache)
    cr = cert_spans('P', n, modes, cb, user,
                    [&](size_t i) {
                      const uint64_t lo = pre_off[msg_idx[i]], hi = pre_off[msg_idx[i] + 1];
                      return hi > lo ? std::string_view(reinterpret_cast<const char *>(preimages + lo), hi - lo) : std::string_view();
                    },
                    [&](size_t i) { return pk + 32 * i; }, [&](size_t i) { return sig + 64 * i; });
  const auto put = [&](queue_sel sel, const hs_queue::req &r) {
    return queue_put_msgs_locked(q, preimages, pre_off, n_msgs, sig, pk, msg_idx, modes, sel, r);
  };
  if (cr) return cert_submit(q, "hs_queue_submit_msgs", std::move(cr), out_ticket, put);
  return queue_submit(q, "hs_queue_submit_msgs", ticket_sink{0, cb, user}, (uint32_t)n, out_ticket,
                      [&](const ticket_sink &s) { return put(queue_sel{nullptr, n}, hs_queue::req{s}); });
}

int hs_queue_poll(hs_queue *q, size_t ticket, int *done, uint32_t *out_bitmap) {
  if (!q || !done || !out_bitmap) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_poll: bad argument");
  std::lock_guard<std::mutex> g(q->mu);
  auto it = q->results.find(ticket);
  if (it == q->results.end()) return fail(q->c, HS_ERR_ARG, "hs_queue_poll: unknown ticket (already read, or consumed by its callback)");
  *done = it->second.done ? 1 : 0;
  if (!it->second.done) return HS_OK;
  const int status = it->second.status;
  memcpy(out_bitmap, it->second.bits.data(), 4 * (size_t)((it->second.n + 31) / 32));
  q->results.erase(it);
  return status;
}

int hs_queue_wait(hs_queue *q, size_t ticket, uint32_t *out_bitmap) {
  if (!q || !out_bitmap) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_wait: bad argument");
  std::unique_lock<std::mutex> lk(q->mu);
  for (;;) {
    auto it = q->results.find(ticket);  // looked up again after every wake-up: submissions may rehash the map
    if (it == q->results.end()) return fail(q->c, HS_ERR_ARG, "hs_queue_wait: unknown ticket (already read, or consumed by its callback)");
    if (it->second.done) {
      const int status = it->second.status;
      memcpy(out_bitmap, it->second.bits.data(), 4 * (size_t)((it->second.n + 31) / 32));
      q->results.erase(it);
      return status;
    }
    q->cv_done.wait(lk);
  }
}

int hs_queue_stats(hs_queue *q, uint64_t out[HS_QUEUE_STATS]) { return queue_read_stats(q, "hs_queue_stats", out, &hs_queue::stats); }

int hs_queue_digest_stats(hs_queue *q, uint64_t out[HS_QUEUE_DIGEST_STATS]) {
  return queue_read_stats(q, "hs_queue_digest_stats", out, &hs_queue::dstats);
}

int hs_queue_cert_cache(hs_queue *q, size_t max_bytes) {
  if (!q) return fail(nullptr, HS_ERR_ARG, "hs_queue_cert_cache: bad argument");
  std::lock_guard<std::mutex> g(q->mu);
  q->cc_max = max_bytes;
  cert_evict_locked(q, max_bytes);
  return HS_OK;
}

int hs_queue_cert_stats(hs_queue *q, uint64_t out[HS_QUEUE_CERT_STATS]) {
  return queue_read_stats(q, "hs_queue_cert_stats", out, &hs_queue::cstats);
}

#define HS_QUEUE_SIG_MAX_ENTRIES (1ull << 26)  // 9.7 GB of table
static int sig_cache_set_locked(hs_queue *q, uint32_t buckets);
int hs_queue_sig_cache(hs_queue *q, size_t entries) {
  if (!q || entries > HS_QUEUE_SIG_MAX_ENTRIES) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_sig_cache: bad argument");
  hs_ctx *c = q->c;
  uint32_t buckets = 0;
  if (entries)
    for (buckets = 1; (size_t)buckets * HS_SIG_WAYS < entries;) buckets <<= 1;
  std::lock_guard<std::mutex> g(c->mu);  // the dispatcher launches only while it holds c->mu
  if (buckets == (q->d_sig ? q->sig_bmask + 1 : 0u)) return HS_OK;
  return sig_cache_set_locked(q, buckets);
}
// Replaces q's signature-cache table by an empty one of `buckets` buckets (0: off), under c->mu.  hs_table_repair empties the cache by
// replacing the table with one of the same size.
static int sig_cache_set_locked(hs_queue *q, uint32_t buckets) {
  hs_ctx *c = q->c;
  HS_CUDA(c, cudaSetDevice(c->device));
  // Drains the queue's streams: no launch that probes the old table survives these lines.  Nor does a batch-lane pass that shares it
  // (hs_queue_sig_share; enqueued under c->mu), and the synchronous calls that share it hold c->mu until their results are back.
  HS_CUDA(c, cudaStreamSynchronize(q->stream));
  HS_CUDA(c, cudaStreamSynchronize(q->bulk_stream));
  if (q->ev_share) HS_CUDA(c, cudaEventSynchronize(q->ev_share));
  if (q->ev_audit) HS_CUDA(c, cudaEventSynchronize(q->ev_audit));  // an audit of the old table (hs_queue_sig_audit, enqueued under c->mu)
  if (!buckets && c->share_q == q) c->share_q = nullptr;  // turning the cache off ends the sharing; a resize keeps it
  q->d_sig.reset();
  {
    std::lock_guard<std::mutex> gq(q->mu);
    q->sig_gen++;
    q->sstats[4] = 0;
  }
  if (!buckets) return HS_OK;
  if (!q->sigc.ctr) {  // first use: the per-slot counters and the bucket mix's key (random per queue)
    uint64_t key[32];
    std::random_device rd;
    for (uint64_t &k : key) k = ((uint64_t)rd() << 32) ^ rd();
    const size_t cb = (size_t)q->cap * HS_SIG_CTRS * 4;
    sig_counters S;
    cudaError_t e = alloc(S.key, sizeof(key));
    if (e == cudaSuccess) e = cudaMemcpy(S.key, key, sizeof(key), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = alloc(S.hctr, cb);
    if (e == cudaSuccess) e = alloc(S.ctr, cb);
    if (e == cudaSuccess) e = cudaMemsetAsync(S.ctr, 0, cb, q->stream);
    if (e != cudaSuccess) return fail(c, HS_ERR_CUDA, "hs_queue_sig_cache", e);  // the cache stays off; a later call starts over
    q->sigc = std::move(S);
  }
  dev_mem<sig_bucket> t;
  const size_t bytes = (size_t)buckets * sizeof(sig_bucket);
  cudaError_t e = alloc(t, bytes);
  if (e == cudaSuccess) e = cudaMemsetAsync(t, 0, bytes, q->stream);  // ahead of every launch that probes it
  if (e == cudaSuccess) e = cudaStreamSynchronize(q->stream);
  if (e != cudaSuccess) return fail(c, e == cudaErrorMemoryAllocation ? HS_ERR_NOMEM : HS_ERR_CUDA, "hs_queue_sig_cache", e);
  q->sig_bmask = buckets - 1;
  q->d_sig = std::move(t);
  return HS_OK;
}

int hs_queue_sig_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_STATS]) {
  return queue_read_stats(q, "hs_queue_sig_stats", out, &hs_queue::sstats);
}

int hs_queue_sig_share(hs_queue *q, int on) {
  if (!q) return fail(nullptr, HS_ERR_ARG, "hs_queue_sig_share: bad argument");
  hs_ctx *c = q->c;
  std::lock_guard<std::mutex> g(c->mu);  // the synchronous calls and the batch lane read c->share_q only while they hold c->mu
  if (!on) {
    if (c->share_q == q) c->share_q = nullptr;
    return HS_OK;
  }
  if (!q->d_sig) return fail(c, HS_ERR_ARG, "hs_queue_sig_share: the queue's signature cache is off");
  if (c->share_q && c->share_q != q) return fail(c, HS_ERR_ARG, "hs_queue_sig_share: another queue of the context shares its cache");
  HS_CUDA(c, cudaSetDevice(c->device));
  if (!q->ev_share) HS_CUDA(c, create(q->ev_share));
  if (!c->share_ctr) {  // first use on the context: the synchronous calls' counters, whole or not at all
    dev_mem<uint32_t> d;
    mapped<uint32_t> h;
    cudaError_t e = alloc(d, 4 * (HS_SIG_CTRS + 1));
    if (e == cudaSuccess) e = alloc(h, 4 * HS_SIG_CTRS);
    if (e != cudaSuccess) return fail(c, HS_ERR_NOMEM, "hs_queue_sig_share", e);
    c->share_ctr = std::move(d);
    c->share_h = std::move(h);
  }
  c->share_q = q;
  return HS_OK;
}

int hs_queue_sig_share_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_SHARE_STATS]) {
  return queue_read_stats(q, "hs_queue_sig_share_stats", out, &hs_queue::shstats);
}

int hs_queue_generic(hs_queue *q, int on) {
  if (!q) return fail(nullptr, HS_ERR_ARG, "hs_queue_generic: bad argument");
  hs_ctx *c = q->c;
  std::lock_guard<std::mutex> g(c->mu);  // the dispatcher reads the option and launches only while it holds c->mu
  if (q->gen_on.load() == (on != 0)) return HS_OK;
  HS_CUDA(c, cudaSetDevice(c->device));
  if (on && !q->gen_bufs.slot.h) {  // first use: the slot list and the descriptor list of the generic launches
    generic_lists G;
    cudaError_t e = alloc(G.slot, (size_t)q->cap * 4);
    if (e == cudaSuccess) e = alloc(G.mlist, (size_t)q->cap * sizeof(qmsg_desc));
    if (e != cudaSuccess)  // the option stays off; a later call starts the first use over
      return fail(c, e == cudaErrorMemoryAllocation ? HS_ERR_NOMEM : HS_ERR_CUDA, "hs_queue_generic", e);
    q->gen_bufs = std::move(G);
  }
  q->gen_on = on != 0;
  if (!on) HS_CUDA(c, cudaStreamSynchronize(q->bulk_stream));  // no generic launch survives this line
  return HS_OK;
}

int hs_queue_generic_stats(hs_queue *q, uint64_t out[HS_QUEUE_GENERIC_STATS]) {
  return queue_read_stats(q, "hs_queue_generic_stats", out, &hs_queue::gstats);
}

#define HS_QUEUE_BATCH_MAX_ITEMS (1u << 24)
#define HS_QUEUE_BATCH_MAX_BYTES (1ull << 30)
int hs_queue_batch(hs_queue *q, size_t max_items, size_t max_bytes) {
  if (!q || (max_items == 0) != (max_bytes == 0) || max_items > HS_QUEUE_BATCH_MAX_ITEMS || max_bytes > HS_QUEUE_BATCH_MAX_BYTES)
    return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_batch: bad argument");
  return lane_configure(q, q->batch, max_items, max_bytes, q->batch_scr, [&](batch_scratch &B, lane_bufs &L, uint64_t, int hi) {
    cudaError_t e = create(L.side, hi);
    for (event_h &ev : B.ev)
      if (e == cudaSuccess) e = create(ev);
    if (e == cudaSuccess) e = alloc(B.dig, (max_bytes / 8 + 1) * 32);  // a preimage costs at least its 8-byte offset
    if (e == cudaSuccess) e = alloc(B.xyz, max_items * 3 * sizeof(fe));
    if (e == cudaSuccess) e = alloc(B.meta, max_items);
    if (e == cudaSuccess) e = alloc(B.vidx, max_items * 4);
    if (e == cudaSuccess) e = alloc(B.miss, max_items * 4);
    if (e == cudaSuccess) e = alloc(B.miss_count, 4);
    if (e == cudaSuccess) e = alloc(B.items, (max_items + 31) / 32 * 4);
    if (e == cudaSuccess) e = alloc(B.grej, max_bytes + 16);  // group words of a region fit in max_bytes
    if (e == cudaSuccess) e = alloc(B.counter, 4);
    if (e == cudaSuccess) e = cudaMemset(B.counter, 0, 4);
    if (e == cudaSuccess) e = alloc(B.share_list, max_items * 4);
    if (e == cudaSuccess) e = alloc(B.share_fl, max_items);
    if (e == cudaSuccess) e = alloc(B.share_ctr, 4 * (HS_SIG_CTRS + 1));
    if (e == cudaSuccess) e = alloc(B.share_h, 4 * HS_SIG_CTRS);
    return e;
  });
}

int hs_queue_submit_batch(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                          const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *modes, size_t n_items, size_t n_groups, hs_queue_cb *cb,
                          void *user, size_t *out_ticket) {
  if (!q || !pre_off || !sig || !pk || !msg_idx || !group_idx || n_items == 0 || n_groups == 0 || n_msgs == 0 || n_items > HS_QUEUE_BATCH_MAX_ITEMS ||
      n_groups > UINT32_MAX || n_msgs > UINT32_MAX)
    return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit_batch: bad argument");
  if (!offsets_ok(pre_off, n_msgs) || (pre_off[n_msgs] && !preimages)) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_batch: bad preimage offsets");
  for (size_t i = 0; i < n_items; i++)
    if (msg_idx[i] >= n_msgs || group_idx[i] >= n_groups || (modes && modes[i] > HS_MODE_BATCH_EQ))
      return fail(q->c, HS_ERR_ARG, "hs_queue_submit_batch: index or mode out of range");
  const uint64_t pre_bytes = pre_off[n_msgs];
  const batch_layout B = batch_layout_of(n_msgs, pre_bytes, n_items, n_groups);
  const lane_req r{{0, cb, user}, batch_bits(n_groups, n_items), (uint32_t)n_items, (uint32_t)n_msgs, (uint32_t)n_groups, pre_bytes, B.o_res, B.o_tail, B.size};
  return lane_submit(q, q->batch, "hs_queue_submit_batch", r, out_ticket, [&](uint8_t *a) {
    memcpy(a, pre_off, 8 * (n_msgs + 1));
    if (pre_bytes) memcpy(a + B.o_pre, preimages, pre_bytes);
    memcpy(a + B.o_sig, sig, 64 * n_items);
    memcpy(a + B.o_pk, pk, 32 * n_items);
    memcpy(a + B.o_mi, msg_idx, 4 * n_items);
    memcpy(a + B.o_gi, group_idx, 4 * n_items);
    if (modes) memcpy(a + B.o_mo, modes, n_items);
    else memset(a + B.o_mo, HS_MODE_STRICT, n_items);
  });
}

int hs_queue_batch_stats(hs_queue *q, uint64_t out[HS_QUEUE_BATCH_STATS]) {
  return queue_read_stats(q, "hs_queue_batch_stats", out, &hs_queue::batch, HS_QUEUE_BATCH_STATS);
}

#define HS_QUEUE_EXPLAIN_MAX_RECORDS (1u << 24)
#define HS_QUEUE_EXPLAIN_MAX_BYTES (1ull << 30)
int hs_queue_explain(hs_queue *q, size_t max_records, size_t max_bytes) {
  if (!q || (max_records == 0) != (max_bytes == 0) || max_records > HS_QUEUE_EXPLAIN_MAX_RECORDS || max_bytes > HS_QUEUE_EXPLAIN_MAX_BYTES)
    return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_explain: bad argument");
  return lane_configure(q, q->explain, max_records, max_bytes, q->explain_scr, [](explain_scratch &X, lane_bufs &, uint64_t acap, int) {
    const uint64_t max_reqs = acap / xq_layout_of(1, 0, 0).size + 1;  // regions the arena holds at once
    return alloc(X.list, max_reqs * sizeof(xq_desc));
  });
}

int hs_queue_submit_explain(hs_queue *q, const hs_rec128 *recs, size_t n, hs_queue_cb *cb, void *user, size_t *out_ticket) {
  if (!q || !recs || n == 0 || n > HS_QUEUE_EXPLAIN_MAX_RECORDS) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit_explain: bad argument");
  const xq_layout L = xq_layout_of(n, 0, 0);
  const lane_req r{{0, cb, user}, explain_bits(n), (uint32_t)n, 0, 0, 0, L.o_why, L.o_tail, L.size};
  return lane_submit(q, q->explain, "hs_queue_submit_explain", r, out_ticket, [&](uint8_t *a) { memcpy(a, recs, n * sizeof(hs_rec128)); });
}

int hs_queue_submit_explain_msgs(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig, const uint8_t *pk,
                                 const uint32_t *msg_idx, size_t n, hs_queue_cb *cb, void *user, size_t *out_ticket) {
  if (!q || !pre_off || !sig || !pk || !msg_idx || n == 0 || n > HS_QUEUE_EXPLAIN_MAX_RECORDS || n_msgs == 0 || n_msgs > UINT32_MAX)
    return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_submit_explain_msgs: bad argument");
  if (!offsets_ok(pre_off, n_msgs) || (pre_off[n_msgs] && !preimages) || pre_off[n_msgs] > HS_QUEUE_EXPLAIN_MAX_BYTES)
    return fail(q->c, HS_ERR_ARG, "hs_queue_submit_explain_msgs: bad preimage offsets");
  for (size_t i = 0; i < n; i++)
    if (msg_idx[i] >= n_msgs) return fail(q->c, HS_ERR_ARG, "hs_queue_submit_explain_msgs: message index out of range");
  const uint64_t pre_bytes = pre_off[n_msgs];
  const xq_layout L = xq_layout_of(n, n_msgs, pre_bytes);
  const lane_req r{{0, cb, user}, explain_bits(n), (uint32_t)n, (uint32_t)n_msgs, 0, pre_bytes, L.o_why, L.o_tail, L.size};
  return lane_submit(q, q->explain, "hs_queue_submit_explain_msgs", r, out_ticket, [&](uint8_t *a) {
    for (size_t i = 0; i < n; i++) {
      memcpy(a + 128 * i, sig + 64 * i, 64);
      memcpy(a + 128 * i + 64, pk + 32 * i, 32);
      memset(a + 128 * i + 96, 0, 32);
    }
    memcpy(a + L.o_off, pre_off, 8 * (n_msgs + 1));
    memcpy(a + L.o_mi, msg_idx, 4 * n);
    if (pre_bytes) memcpy(a + L.o_pre, preimages, pre_bytes);
  });
}

int hs_queue_explain_stats(hs_queue *q, uint64_t out[HS_QUEUE_EXPLAIN_STATS]) {
  return queue_read_stats(q, "hs_queue_explain_stats", out, &hs_queue::explain, HS_QUEUE_EXPLAIN_STATS);
}

void hs_queue_destroy(hs_queue *q) {
  if (!q) return;
  {
    std::lock_guard<std::mutex> g(q->c->mu);  // ends the sharing (hs_queue_sig_share): later synchronous calls run without the table
    if (q->c->share_q == q) q->c->share_q = nullptr;
  }
  {
    std::lock_guard<std::mutex> l(q->c->scrub.m);  // a scrub tick auditing q's cache (hs_scrub_sig_cache) holds it until it is done
    if (q->c->scrub.sig_q == q) q->c->scrub.sig_q = nullptr;
  }
  {
    std::lock_guard<std::mutex> g(q->c->queues_mu);
    auto &v = q->c->queues;
    for (size_t i = 0; i < v.size(); i++)
      if (v[i] == q) {
        v.erase(v.begin() + (long)i);
        break;
      }
  }
  queue_free(q);
}

}  // extern "C"

// ================================================================================================ known-answer self-test (hs_self_test)
// Drives the existing kernels on private scratch, at the context's base window and a chosen per-key window, and compares their
// verdicts, digests, keys and signatures with answers compiled into the library.  Nothing of the context is written but its launch
// counter and its last-error text: the scratch key tables, the hash table, the queue ring, the signature table and the streams are
// the call's own and are released before it returns.

#define HS_SELFTEST_MAX_RECORDS 4096u
#define HS_SELFTEST_FIN_GROUP 4  // records per thread of k_verify_finish, as run_verify picks for small passes

namespace {
// The records of one run: those with a 32-byte message (every path) and every record as a variable-length message (the var-length
// path), each with its expected verdicts (bit 0 strict, bit 1 batch-eq) and its name for the error text.
struct st_set {
  std::vector<hs_rec128> r32;
  std::vector<uint8_t> e32;
  std::vector<std::string> n32;
  std::vector<uint8_t> sig, pk, msgs;
  std::vector<uint64_t> off{0};
  std::vector<uint8_t> ev;
  std::vector<std::string> nv;
  void add(const std::string &name, const uint8_t *s, const uint8_t *k, const uint8_t *m, size_t len, uint8_t expect) {
    if (len == 32) {
      hs_rec128 r;
      memcpy(r.sig, s, 64);
      memcpy(r.pk, k, 32);
      memcpy(r.msg, m, 32);
      r32.push_back(r);
      e32.push_back(expect);
      n32.push_back(name);
    }
    sig.insert(sig.end(), s, s + 64);
    pk.insert(pk.end(), k, k + 32);
    msgs.insert(msgs.end(), m, m + len);
    off.push_back(msgs.size());
    ev.push_back(expect);
    nv.push_back(name);
  }
};
// Failed paths, and the first mismatch found.
struct st_result {
  uint32_t failed = 0;
  std::string first;
  void mismatch(uint32_t bit, const std::string &what) {
    if (!failed) first = "hs_self_test: " + what;
    failed |= bit;
  }
};
// got(i): record i's verdict bits; checked bits: 3, or 1 << mode[i] when mode is given (k_verify_finish_modes).
template <class Got>
void st_compare(st_result &R, uint32_t bit, const char *path, const std::vector<std::string> &names, const std::vector<uint8_t> &expect,
                const uint8_t *mode, Got got) {
  for (size_t i = 0; i < expect.size(); i++) {
    const uint32_t mask = mode ? 1u << mode[i] : 3u, g = got(i) & mask, want = expect[i] & mask;
    if (g == want) continue;
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s (record %zu): got strict=%s batch_eq=%s, expected strict=%s batch_eq=%s", path, names[i].c_str(), i,
             (mask & 1) ? ((g & 1) ? "1" : "0") : "-", (mask & 2) ? ((g & 2) ? "1" : "0") : "-", (mask & 1) ? ((want & 1) ? "1" : "0") : "-",
             (mask & 2) ? ((want & 2) ? "1" : "0") : "-");
    R.mismatch(bit, buf);
    return;
  }
}
// Waits for the private streams when it goes out of scope: declared after the buffers a helper launches on, it keeps every return path
// from releasing memory that work in flight still uses.
struct st_drain {
  cudaStream_t a, b;
  ~st_drain() {
    cudaStreamSynchronize(a);
    if (b) cudaStreamSynchronize(b);
  }
};
uint8_t st_flag_bits(uint8_t fl) { return ((fl & HS_F_STRICT) ? 1u : 0u) | ((fl & HS_F_EQ) ? 2u : 0u); }
uint8_t st_bitmap_bits(const std::vector<uint32_t> &strict, const std::vector<uint32_t> &eq, size_t i) {
  return (uint8_t)(((strict[i >> 5] >> (i & 31)) & 1u) | (((eq[i >> 5] >> (i & 31)) & 1u) << 1));
}
}  // namespace

// Device results of one path, read back on the private stream.
static int st_read(hs_ctx *c, cudaStream_t st, void *dst, const void *src, size_t bytes) {
  HS_CUDA(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
  HS_CUDA(c, cudaStreamSynchronize(st));
  return HS_OK;
}

// The three Digest kernels over the SHA-512 known answers, and k_keygen / k_sign_digests over the seeded keys, each through the launch
// the product uses.  Keygen and signing read only the base-point window of the context's cp, which the self-test's cp shares.
static int st_digest_and_sign_paths(hs_ctx *c, cudaStream_t st, st_result &R) {
  const size_t n = HS_ST_N_DIGEST_KATS;
  std::vector<uint64_t> off(n + 1);
  for (size_t i = 0; i < n; i++) off[i] = hs_st_digest_kats[i].off;
  off[n] = HS_ST_KAT_MSG_BYTES;
  std::vector<uint8_t> seeds(32 * (HS_ST_N_SEEDS + 1)), pks(32 * HS_ST_N_SEEDS), dig(32 * HS_ST_N_SIGNATURES);
  std::vector<uint32_t> key_idx(HS_ST_N_SIGNATURES);
  memcpy(seeds.data(), hs_st_seeds, 32 * HS_ST_N_SEEDS);
  memcpy(seeds.data() + 32 * HS_ST_N_SEEDS, hs_st_tv1_seed, 32);
  memcpy(pks.data(), hs_st_seed_pks, 32 * HS_ST_N_SEEDS);
  for (size_t i = 0; i < HS_ST_N_SIGNATURES; i++) {
    memcpy(dig.data() + 32 * i, hs_st_signatures[i].digest, 32);
    key_idx[i] = hs_st_signatures[i].key;
  }
  dev_buf buf;
  h2d_stage S;
  const size_t s_off = S.add(off.data(), off.size() * 8), s_data = S.add(hs_st_kat_msgs, HS_ST_KAT_MSG_BYTES, 8), s_out = S.add(nullptr, 32 * n),
               s_seed = S.add(seeds.data(), seeds.size()), s_pk = S.add(pks.data(), pks.size()), s_ki = S.add(key_idx.data(), key_idx.size() * 4),
               s_dig = S.add(dig.data(), dig.size()), s_res = S.add(nullptr, 64 * (HS_ST_N_SEEDS + 1 + HS_ST_N_SIGNATURES));
  HS_TRY(S.upload(c, buf, st));
  const st_drain drain{st, nullptr};
  uint32_t *d_out = (uint32_t *)S.ptr(s_out);
  std::vector<uint8_t> got(32 * n);
  auto check_digests = [&](uint32_t bit, const char *path, size_t i) {
    if (memcmp(got.data() + 32 * i, hs_st_digest_kats[i].digest, 32) == 0) return;
    char b[160];
    snprintf(b, sizeof b, "%s: digest known answer %zu (%u bytes): wrong Digest", path, i, hs_st_digest_kats[i].len);
    R.mismatch(bit, b);
  };
  HS_TRY(hs_digest32_dev(c, S.ptr(s_data), S.ptr(s_off), n, d_out, st));
  HS_TRY(st_read(c, st, got.data(), d_out, 32 * n));
  for (size_t i = 0; i < n; i++) check_digests(HS_SELFTEST_DIGEST, "k_digest32", i);
  HS_CUDA(c, cudaMemsetAsync(d_out, 0, 32 * n, st));
  HS_TRY(launch_digest_long(c, S.ptr(s_data), (const uint64_t *)S.ptr(s_off), n, d_out, st));
  HS_TRY(st_read(c, st, got.data(), d_out, 32 * n));
  for (size_t i = 0; i < n; i++) check_digests(HS_SELFTEST_DIGEST_LONG, "k_digest32_long", i);
  // k_digest32_fixed takes 16-byte aligned messages of at least one full block, one launch per length
  for (size_t i = 0; i < n; i++) {
    const hs_st_digest_kat &k = hs_st_digest_kats[i];
    if (k.len < 128 || (k.len & 15)) continue;
    dev_mem<uint8_t> m;
    HS_CUDA(c, alloc(m, k.len));
    const st_drain drain_m{st, nullptr};
    HS_CUDA(c, cudaMemcpyAsync(m, hs_st_kat_msgs + k.off, k.len, cudaMemcpyHostToDevice, st));
    HS_CUDA(c, cudaMemsetAsync(d_out, 0, 32, st));
    HS_TRY(launch_digest_fixed(c, m, k.len, 1, d_out, st));
    HS_TRY(st_read(c, st, got.data() + 32 * i, d_out, 32));
    check_digests(HS_SELFTEST_DIGEST_FIXED, "k_digest32_fixed", i);
  }
  // keys of the seeded test keys and RFC 8032 TEST 1, then the signatures of 32-byte digests
  uint8_t *d_res = S.ptr(s_res);
  HS_TRY(hs_keygen_batch_dev(c, S.ptr(s_seed), HS_ST_N_SEEDS + 1, d_res, st));
  HS_TRY(hs_sign_digests_dev(c, S.ptr(s_seed), S.ptr(s_pk), HS_ST_N_SEEDS, S.ptr(s_ki), S.ptr(s_dig), HS_ST_N_SIGNATURES,
                             d_res + 32 * (HS_ST_N_SEEDS + 1), st));
  std::vector<uint8_t> res(32 * (HS_ST_N_SEEDS + 1) + 64 * HS_ST_N_SIGNATURES);
  HS_TRY(st_read(c, st, res.data(), d_res, res.size()));
  for (size_t i = 0; i <= HS_ST_N_SEEDS; i++) {
    const uint8_t *want = i < HS_ST_N_SEEDS ? hs_st_seed_pks[i] : hs_st_tv1_pk;
    if (memcmp(res.data() + 32 * i, want, 32) == 0) continue;
    R.mismatch(HS_SELFTEST_SIGN, i < HS_ST_N_SEEDS ? "k_keygen: seeded key " + std::to_string(i) + ": wrong public key"
                                                   : std::string("k_keygen: RFC 8032 TEST 1: wrong public key"));
    break;
  }
  for (size_t i = 0; i < HS_ST_N_SIGNATURES; i++) {
    if (memcmp(res.data() + 32 * (HS_ST_N_SEEDS + 1) + 64 * i, hs_st_signatures[i].sig, 64) == 0) continue;
    R.mismatch(HS_SELFTEST_SIGN, "k_sign_digests: signature " + std::to_string(i) + ": wrong signature");
    break;
  }
  return HS_OK;
}

// The scratch per-key tables: the set's distinct keys, built by k_build_comb at window cp.wa like a registration, and a hash table built
// on the host over every key but `foreign`, whose records therefore miss k_key_lookup and take the side-stream generic pass.
struct st_keys {
  std::vector<uint8_t> pks;  // distinct keys, 32 bytes each, in first-seen order
  std::unordered_map<std::string, uint32_t> index;
  key_index h_index;
  key_store K;
  uint32_t idx(const uint8_t *pk) const { return index.at(std::string((const char *)pk, 32)); }
};
static int st_build_keys(hs_ctx *c, const st_set &T, const comb_params &cp, st_keys &KS, pass_tables &K, cudaStream_t st) {
  const size_t n = KS.pks.size() / 32;
  const uint32_t foreign = T.r32.empty() ? HS_NO_KEY : KS.idx(T.r32[0].pk);
  KS.h_index.reset(n);
  KS.h_index.build(KS.pks.data(), n, [foreign](size_t i) { return i != foreign; });
  const cudaError_t e = make_key_store(KS.K, n, KS.h_index.slots.size(), cp.wa, st);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(c, HS_ERR_NOMEM, "hs_self_test: the scratch key tables do not fit in device memory", e);
  }
  HS_CUDA(c, cudaMemcpyAsync(KS.K.pks, KS.pks.data(), n * 32, cudaMemcpyHostToDevice, st));
  HS_CUDA(c, cudaMemcpyAsync(KS.K.slots, KS.h_index.slots.data(), KS.h_index.slots.size() * 4, cudaMemcpyHostToDevice, st));
  HS_TRY(launch_build(c, KS.K.pks, nullptr, n, 1, cp.wa, cp.na, KS.K.atables, KS.K.key_flags, st));
  K = store_tables(KS.K, KS.h_index, n, comb_table_entries(cp.wa), cp);
  return HS_OK;
}

// Every verify path over the set: the throughput passes (k_verify_main + k_verify_finish in both modes, k_verify_finish_modes) and the
// queue kernels on a private mapped ring.
static int st_verify_paths(hs_ctx *c, const st_set &T, const st_keys &KS, const pass_tables &K, cudaStream_t st, cudaStream_t side,
                           st_result &R) {
  const size_t n = T.r32.size(), nv = T.ev.size(), nmax = std::max(n, nv);
  std::vector<uint32_t> vidx(n);
  std::vector<uint8_t> modes(n);
  for (size_t i = 0; i < n; i++) {
    vidx[i] = KS.idx(T.r32[i].pk);
    modes[i] = (uint8_t)(i & 1);
  }
  const size_t words = (nmax + 31) / 32;
  dev_buf buf;
  h2d_stage S;
  const size_t s_recs = S.add(T.r32.data(), n * sizeof(hs_rec128)), s_vidx = S.add(vidx.data(), n * 4), s_modes = S.add(modes.data(), n),
               s_sig = S.add(T.sig.data(), nv * 64), s_pk = S.add(T.pk.data(), nv * 32), s_off = S.add(T.off.data(), (nv + 1) * 8),
               s_msg = S.add(T.msgs.data(), T.msgs.size(), 8);
  HS_TRY(S.upload(c, buf, st));
  dev_mem<fe> xyz;
  dev_mem<uint8_t> meta;
  dev_mem<uint32_t> lk, bm;  // lk: the lookup's indices, misses and miss count; bm: the strict, batch-eq and mixed-mode bitmaps
  HS_CUDA(c, alloc(xyz, nmax * 3 * sizeof(fe)));
  HS_CUDA(c, alloc(meta, nmax));
  HS_CUDA(c, alloc(lk, 2 * n * 4 + 4));
  HS_CUDA(c, alloc(bm, 3 * words * 4));
  event_h ev_side[2];
  for (event_h &ev : ev_side) HS_CUDA(c, create(ev));
  const st_drain drain{st, side};
  const pass_scratch PS{xyz, meta, lk, lk + n, lk + 2 * n, side, {ev_side[0], ev_side[1]}, nullptr};
  std::vector<uint32_t> strict(words), eq(words), mixed(words);
  // one main phase, then the finish kernel in both modes (and with mixed mode bytes), the bitmaps compared with the expectations
  auto pass = [&](uint32_t bit, const char *path, in_layout L, bool var, bool committee, bool indexed, uint32_t modes_bit) -> int {
    const size_t cnt = var ? nv : n;
    if (cnt == 0) return HS_OK;
    HS_CUDA(c, cudaMemsetAsync(bm, 0, 3 * words * 4, st));
    HS_TRY(launch_main(c, L, cnt, committee, indexed, K, PS, st, [](bool) { return HS_OK; }));
    HS_TRY(launch_finish(c, L, cnt, PS.xyz, PS.meta, HS_MODE_STRICT, nullptr, bm, peer_route{}, HS_SELFTEST_FIN_GROUP, st));
    HS_TRY(launch_finish(c, L, cnt, PS.xyz, PS.meta, HS_MODE_BATCH_EQ, nullptr, bm + words, peer_route{}, HS_SELFTEST_FIN_GROUP, st));
    if (modes_bit)
      HS_TRY(launch_finish(c, L, cnt, PS.xyz, PS.meta, HS_MODE_STRICT, S.ptr(s_modes), bm + 2 * words, peer_route{}, HS_SELFTEST_FIN_GROUP, st));
    HS_CUDA(c, cudaMemcpyAsync(strict.data(), bm, words * 4, cudaMemcpyDeviceToHost, st));
    HS_CUDA(c, cudaMemcpyAsync(eq.data(), bm + words, words * 4, cudaMemcpyDeviceToHost, st));
    HS_TRY(st_read(c, st, mixed.data(), bm + 2 * words, words * 4));
    st_compare(R, bit, path, var ? T.nv : T.n32, var ? T.ev : T.e32, nullptr, [&](size_t i) { return st_bitmap_bits(strict, eq, i); });
    if (modes_bit)
      st_compare(R, modes_bit, "k_verify_finish_modes", T.n32, T.e32, modes.data(),
                 [&](size_t i) { return (uint8_t)(((mixed[i >> 5] >> (i & 31)) & 1u) << modes[i]); });
    return HS_OK;
  };
  const uint8_t *recs = S.ptr(s_recs);
  HS_TRY(pass(HS_SELFTEST_GENERIC, "k_verify_main<generic> (packed records)", layout_rec128(recs), false, false, false, 0));
  HS_TRY(pass(HS_SELFTEST_VAR, "k_verify_main<generic> (variable-length messages)",
              in_layout{S.ptr(s_sig), 64, S.ptr(s_pk), 32, nullptr, S.ptr(s_msg), 0, nullptr, (const uint64_t *)S.ptr(s_off), 0, 0}, true, false, false, 0));
  HS_TRY(pass(HS_SELFTEST_COMMITTEE, "k_verify_main<committee> (committee indices)",
              in_layout{recs, 128, nullptr, 0, (const uint32_t *)S.ptr(s_vidx), recs + 96, 128, nullptr, nullptr, 32, 0}, false, true, true,
              HS_SELFTEST_MODES));
  HS_TRY(pass(HS_SELFTEST_LOOKUP, "k_key_lookup + k_verify_main<committee> + side pass", layout_rec128(recs), false, true, false, 0));
  if (n == 0) return HS_OK;

  // the queue kernels: one request of n records in slot 0 of a private mapped ring
  uint32_t cap = HS_SMALL_MAX;
  while (cap < n) cap <<= 1;
  const uint32_t mask = cap - 1, buckets = std::max(cap / 2, 16u);
  ring_bufs ring;
  mapped<uint8_t> pk;
  mapped<uint32_t> slot, hctr;
  dev_mem<uint32_t> ctr;
  dev_mem<sig_bucket> table;
  dev_mem<uint64_t> key;
  HS_CUDA(c, make_ring(ring, cap, st));
  HS_CUDA(c, alloc(pk, (size_t)cap * 32));
  HS_CUDA(c, alloc(slot, (size_t)cap * 4));
  HS_CUDA(c, alloc(hctr, (size_t)cap * 4 * HS_SIG_CTRS));
  HS_CUDA(c, alloc(ctr, (size_t)cap * 4 * HS_SIG_CTRS));
  HS_CUDA(c, alloc(table, (size_t)buckets * sizeof(sig_bucket)));
  HS_CUDA(c, alloc(key, 32 * 8));
  const st_drain drain_ring{st, nullptr};
  uint64_t kh[32];
  uint64_t z = 0x243f6a8885a308d3ull;  // any fixed key: the table is private and short-lived
  for (uint64_t &k : kh) k = (z += 0x9e3779b97f4a7c15ull) ^ (z >> 29);
  HS_CUDA(c, cudaMemcpyAsync(key, kh, sizeof kh, cudaMemcpyHostToDevice, st));
  HS_CUDA(c, cudaMemsetAsync(ctr, 0, (size_t)cap * 4 * HS_SIG_CTRS, st));
  memset(ring.recs.h, 0, (size_t)cap * sizeof(small_rec));
  for (uint32_t i = 0; i < n; i++) {
    memcpy(ring.recs.h[i].sig, T.r32[i].sig, 64);
    memcpy(ring.recs.h[i].msg, T.r32[i].msg, 32);
    ring.recs.h[i].vidx = vidx[i];
    ring.recs.h[i].req = 0;
    ring.recs.h[i].req_n = (uint32_t)n;
    memcpy(pk.h + 32 * (size_t)i, T.r32[i].pk, 32);
    slot.h[i] = i;
  }
  uint32_t seq = 0;
  // launch(seq) enqueues one kernel over the request; its completion word and its records' flags are then compared
  auto queue_pass = [&](uint32_t bit, const char *path, auto launch) -> int {
    memset(ring.flags.h, 0, cap);
    HS_CUDA(c, launch(++seq));
    HS_CUDA(c, cudaStreamSynchronize(st));
    if (((volatile uint32_t *)ring.done.h)[0] != seq) {
      R.mismatch(bit, std::string(path) + ": the request did not complete");
      return HS_OK;
    }
    st_compare(R, bit, path, T.n32, T.e32, nullptr, [&](size_t i) { return st_flag_bits(ring.flags.h[i]); });
    return HS_OK;
  };
  // k_verify_small and k_verify_bulk without the signature cache, then k_queue_generic, then the two with the cache, each twice on an
  // empty table: the first run probes, misses and inserts, the second answers from it
  const sig_cache_dev sc{table, key, buckets - 1, ctr, hctr.d};
  static const uint32_t bits[2][2] = {{HS_SELFTEST_SMALL, HS_SELFTEST_BULK}, {HS_SELFTEST_SMALL_CACHE, HS_SELFTEST_BULK_CACHE}};
  for (int cached = 0; cached < 2; cached++) {
    for (int bulk = 0; bulk < 2; bulk++) {
      if (cached) HS_CUDA(c, cudaMemsetAsync(table, 0, (size_t)buckets * sizeof(sig_bucket), st));
      const std::string kernel = bulk ? "k_verify_bulk" : "k_verify_small";
      for (int run = 0; run <= cached; run++) {
        const std::string path = cached ? kernel + (run ? "<cache> (cache filled)" : "<cache> (empty cache)") : kernel;
        HS_TRY(queue_pass(bits[cached][bulk], path.c_str(), [&](uint32_t s) {
          return launch_ring_verify(c, ring, mask, 0, (uint32_t)n, bulk, K.C, K.cp, cached ? sc : sig_cache_dev{}, s, st);
        }));
      }
    }
    if (!cached)
      HS_TRY(queue_pass(HS_SELFTEST_QUEUE_GENERIC, "k_queue_generic",
                        [&](uint32_t s) { return launch_queue_generic(c, ring, pk.d, slot.d, mask, 0, (uint32_t)n, K.cp, s, st); }));
  }
  return HS_OK;
}

// k_queue_digests over the SHA-512 known answers: one request of one record per preimage on a private ring; each record's msg field
// must receive its preimage's Digest.
static int st_queue_digest_path(hs_ctx *c, cudaStream_t st, st_result &R) {
  const uint32_t m = HS_ST_N_DIGEST_KATS, n = HS_ST_N_DIGEST_KATS, cap = HS_SMALL_MAX;
  const uint64_t bytes = qmsg_bytes(m, n, HS_ST_KAT_MSG_BYTES);
  mapped<uint8_t> arena;
  mapped<qmsg_desc> list;
  ring_bufs ring;
  dev_mem<uint8_t> stage;
  dev_mem<uint32_t> digs;
  HS_CUDA(c, alloc(arena, bytes));
  HS_CUDA(c, alloc(list, sizeof(qmsg_desc)));
  HS_CUDA(c, make_ring(ring, cap, st));
  HS_CUDA(c, alloc(stage, bytes));
  HS_CUDA(c, alloc(digs, bytes * 4));
  const st_drain drain{st, nullptr};
  memset(arena.h, 0, bytes);
  memset(ring.recs.h, 0, (size_t)cap * sizeof(small_rec));
  uint64_t *off = reinterpret_cast<uint64_t *>(arena.h.get());
  uint32_t *msg_idx = reinterpret_cast<uint32_t *>(arena.h + 8 * ((size_t)m + 1));
  for (uint32_t i = 0; i < m; i++) {
    off[i] = hs_st_digest_kats[i].off;
    msg_idx[i] = i;
  }
  off[m] = HS_ST_KAT_MSG_BYTES;
  memcpy(arena.h + qmsg_o_pre(m, n), hs_st_kat_msgs, HS_ST_KAT_MSG_BYTES);
  *list.h = qmsg_desc{0, m, n, 0, HS_ST_KAT_MSG_BYTES, {0, 0, 0}};
  HS_CUDA(c, launch_queue_digests(c, ring, list.d, cap - 1, 0, 1, arena.d, stage, digs, st));
  HS_CUDA(c, cudaStreamSynchronize(st));
  for (uint32_t i = 0; i < n; i++) {
    if (memcmp(ring.recs.h[i].msg, hs_st_digest_kats[i].digest, 32) == 0) continue;
    R.mismatch(HS_SELFTEST_QUEUE_DIGESTS, "k_queue_digests: digest known answer " + std::to_string(i) + ": wrong Digest");
    break;
  }
  return HS_OK;
}

static int self_test_locked(hs_ctx *c, int key_bits, const hs_rec128 *recs, const uint8_t *expect, size_t n, uint32_t *out_failed) {
  HS_CUDA(c, cudaSetDevice(c->device));
  st_set T;
  if (!recs) {
    for (const hs_st_vector &v : hs_st_vectors) T.add(v.name, v.sig, v.pk, hs_st_vec_msgs + v.msg_off, v.msg_len, v.expect);
  } else {
    for (size_t i = 0; i < n; i++) T.add("caller record " + std::to_string(i), recs[i].sig, recs[i].pk, recs[i].msg, 32, expect[i]);
  }
  st_keys KS;
  for (size_t i = 0; i < T.ev.size(); i++) {
    const std::string k((const char *)T.pk.data() + 32 * i, 32);
    if (KS.index.emplace(k, (uint32_t)(KS.pks.size() / 32)).second) KS.pks.insert(KS.pks.end(), k.begin(), k.end());
  }
  int wa = key_bits;
  if (wa == 0 && c->keys.atables) wa = c->cp.wa;  // the registered committee's window, or the key cache's
  if (wa == 0) {                                  // neither: the window registering these keys would get now
    size_t capk = 0;
    HS_TRY(committee_geometry(c, KS.pks.size() / 32, capk, wa));
  }
  comb_params cp = c->cp;
  set_window(cp, true, wa);
  if (cp.na + cp.nb > HS_MAX_DIGITS) return fail(c, HS_ERR_ARG, "hs_self_test: window combination exceeds HS_MAX_DIGITS");
  stream_h st, side;  // private: the work of this call only (the drain below waits for both before any scratch is released)
  int lo = 0, hi = 0;
  HS_CUDA(c, cudaDeviceGetStreamPriorityRange(&lo, &hi));
  HS_CUDA(c, create(st));
  HS_CUDA(c, create(side, hi));
  st_result R;
  {
    const st_drain drain{st, side};
    pass_tables K;
    HS_TRY(st_build_keys(c, T, cp, KS, K, st));
    if (!recs) {
      HS_TRY(st_digest_and_sign_paths(c, st, R));
      HS_TRY(st_queue_digest_path(c, st, R));
    }
    HS_TRY(st_verify_paths(c, T, KS, K, st, side, R));
  }
  HS_CUDA(c, cudaGetLastError());
  *out_failed = R.failed;
  return R.failed ? fail(c, HS_ERR_SELFTEST, R.first.c_str()) : HS_OK;
}

extern "C" int hs_self_test(hs_ctx *c, int key_bits, const hs_rec128 *recs, const uint8_t *expect, size_t n, uint32_t *out_failed_paths) {
  if (out_failed_paths) *out_failed_paths = 0;
  if (!c || !out_failed_paths || (key_bits != 0 && (key_bits < 8 || key_bits > 17))) return fail(c, HS_ERR_ARG, "hs_self_test: bad argument");
  if (recs ? (!expect || n == 0 || n > HS_SELFTEST_MAX_RECORDS) : (expect || n != 0))
    return fail(c, HS_ERR_ARG, "hs_self_test: caller records need expectations and 1 .. 4096 records; the built-in set takes none");
  for (size_t i = 0; recs && i < n; i++)
    if (expect[i] > 3) return fail(c, HS_ERR_ARG, "hs_self_test: an expectation byte uses bits other than 0 and 1");
  std::lock_guard<std::mutex> g(c->mu);
  return self_test_locked(c, key_bits, recs, expect, n, out_failed_paths);
}

// ---- audit of the live key tables (hs_table_audit)
extern "C" size_t hs_key_slots(const hs_ctx *c) { return (c && has_key_tables(c)) ? c->n_keys : 0; }

// The message for the first finding: audit_key() decoded, with the slot's classes for a finding about the slot itself.
static std::string audit_message(uint64_t first, size_t n_slots, const uint32_t *bits) {
  const uint64_t code = first >> 32;
  const uint32_t wfield = (uint32_t)(first >> 26) & 63u, entry = (uint32_t)first & ((1u << 26) - 1);
  const std::string at = wfield ? ": window " + std::to_string(wfield - 1) + ", entry " + std::to_string(entry) : std::string();
  if (code == 0) return "hs_table_audit: base-point table" + at + " is not the multiple of B it must hold (BASE)";
  if (code > n_slots) return "hs_table_audit: a device hash-table entry names a slot past the " + std::to_string(n_slots) + " in use (LOOKUP)";
  const size_t s = (size_t)code - 1;
  if (wfield) return "hs_table_audit: slot " + std::to_string(s) + ": comb table" + at + " is not the multiple of -A it must hold (TABLE)";
  std::string m = "hs_table_audit: slot " + std::to_string(s) + ":";
  if (bits[2 + s] & HS_AUDIT_KEY) m += " stored key bytes or liveness differ from the expectation (KEY);";
  if (bits[2 + s] & HS_AUDIT_FLAG) m += " device flag byte disagrees with liveness and decompression (FLAG);";
  if (bits[2 + s] & HS_AUDIT_LOOKUP) m += " device hash table does not map its key bytes to a live slot with them (LOOKUP);";
  m.pop_back();
  return m;
}

// Entries [first, first + count) of the base-point table, count > 0 (the range form of k_table_audit).
struct base_range {
  uint64_t first, count;
};
// k_table_audit over n_tables tables on `stream`: tables 0 .. n_tables - 1, or with d_slots the listed slots' (auditable and findings by
// list position), or with `range` that range of the base-point table.  auditable: nullable for the base-point table.
static int launch_table_audit(hs_ctx *c, cudaStream_t stream, const ge_niels *tables, const uint32_t *d_slots, size_t n_tables, size_t entries,
                              int W, int n_windows, const uint8_t *pks, const uint8_t *auditable, const audit_out &O,
                              const base_range *range = nullptr, const audit_wins *wins = nullptr) {
  const uint64_t stride = comb_window_stride(W), runs = (stride + 31) / 32;
  const auto run_of = [&](uint64_t e) { return e / stride * runs + e % stride / 32; };
  const uint64_t warps = range ? run_of(range->first + range->count - 1) - run_of(range->first) + 1 : (uint64_t)n_tables * n_windows * runs;
  const unsigned blocks = (unsigned)((warps + HS_AUDIT_WARPS - 1) / HS_AUDIT_WARPS);
  const auto launch = [&](auto listed, auto... args) {
    k_table_audit<decltype(listed)::value><<<blocks, 32 * HS_AUDIT_WARPS, 0, stream>>>(tables, args...);
  };
  if (wins) {  // the same forms with the window findings (hs_table_mend)
    if (range) launch(std::false_type{}, range->first, range->count, W, n_windows, O, *wins);
    else if (d_slots) launch(std::true_type{}, d_slots, n_tables, entries, W, n_windows, pks, auditable, O, *wins);
    else launch(std::false_type{}, d_slots, n_tables, entries, W, n_windows, pks, auditable, O, *wins);
  } else if (range) launch(std::false_type{}, range->first, range->count, W, n_windows, O);
  else if (d_slots) launch(std::true_type{}, d_slots, n_tables, entries, W, n_windows, pks, auditable, O);
  else launch(std::false_type{}, d_slots, n_tables, entries, W, n_windows, pks, auditable, O);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}

// k_slot_audit over the slots and hash entries of T on `stream`: the KEY / FLAG / LOOKUP checks against the liveness mirror `live` and
// the caller's map (expect_pks / expect_live, nullable), writing `auditable` for k_table_audit.
static int launch_slot_audit(hs_ctx *c, cudaStream_t stream, const key_table &T, const uint8_t *key_flags, const uint8_t *live,
                             const uint8_t *expect_pks, const uint32_t *expect_live, uint8_t *auditable, const audit_out &O) {
  k_slot_audit<<<blocks_for((size_t)T.n_keys + (size_t)T.mask + 1, 256), 256, 0, stream>>>(T, key_flags, live, expect_pks, expect_live,
                                                                                          (expect_pks || expect_live) ? 1 : 0, auditable, O);
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return HS_OK;
}

// The audit's private stream of the lowest priority and its event, created on first use.
static int audit_stream(hs_ctx *c) {
  audit_state &A = c->audit;
  if (!A.stream) {
    int lo = 0, hi = 0;
    HS_CUDA(c, cudaDeviceGetStreamPriorityRange(&lo, &hi));
    HS_CUDA(c, create(A.stream, lo));
    HS_CUDA(c, create(A.done));
  }
  return HS_OK;
}
// One complete audit: enqueued under c->mu by audit_enqueue_locked, then waited for and read back without it by audit_collect.  Its
// caller holds audit_mu, so the audit's stream, event and scratch are its own.
struct audit_run {
  uint64_t gen = 0;              // key_gen when the kernels were enqueued
  size_t n_slots = 0;
  const uint8_t *d_res = nullptr;
  std::vector<uint8_t> res;      // the first finding's audit_key() (8 bytes), then bits[2 + n_slots], then the window findings
  // With the window findings (hs_table_mend's audits): the audit_wins bits of the key tables from bit 0 (table t's row at t (na + 1)),
  // those of the base-point table from word base_word (row 0, nb + 1 bits).  win_words == 0: none.
  int na = 0, nb = 0;
  size_t base_word = 0, win_words = 0;
  uint64_t first() const {
    uint64_t f;
    memcpy(&f, res.data(), 8);
    return f;
  }
  const uint32_t *bits() const { return reinterpret_cast<const uint32_t *>(res.data() + 8); }
  uint32_t failed() const {
    uint32_t f = (bits()[0] ? HS_AUDIT_BASE : 0u) | bits()[1];
    for (size_t s = 0; s < n_slots; s++) f |= bits()[2 + s];
    return f;
  }
  uint32_t *wins() { return reinterpret_cast<uint32_t *>(res.data() + 8) + 2 + n_slots; }
  const uint32_t *wins() const { return bits() + 2 + n_slots; }
  bool win_bit(uint64_t b) const { return (wins()[b >> 5] >> (b & 31)) & 1u; }
  bool key_win(size_t t, int i) const { return win_bit((uint64_t)t * (na + 1) + i); }  // i == na: the anchor failed
  bool base_win(int i) const { return win_bit(32 * (uint64_t)base_word + i); }
  // Sizes the window findings for n_keys key tables and the base-point table at c's geometry.
  void size_windows(const comb_params &cp, size_t n_keys) {
    na = cp.na;
    nb = cp.nb;
    base_word = (n_keys * (size_t)(na + 1) + 31) / 32;
    win_words = base_word + (nb + 1 + 31) / 32;
  }
};
// Part of an audit (a scrub tick): the KEY / FLAG / LOOKUP checks of every slot and hash entry as the complete audit runs them (a
// thread each), the comb tables of the slots in `tables` only, and entries [base_first, base_first + base_count) of the base-point table.
// Findings land at the slots' own bits; the first-finding key names a slot relative to its run and is not read.
struct audit_slice {
  std::vector<std::pair<size_t, size_t>> tables;  // [begin, end) runs of slots
  uint64_t base_first = 0, base_count = 0;
};
// Checks the arguments, snapshots the slots and their liveness, uploads and enqueues: the complete audit, or with `slice` that part.
// Nothing here waits for a kernel.
// windows: the WINDOWS forms, with the window findings in r (hs_table_mend and a scrub that mends).
static int audit_enqueue_locked(hs_ctx *c, const char *entry, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots,
                                audit_run &r, const audit_slice *slice = nullptr, bool windows = false) {
  audit_state &A = c->audit;
  HS_CUDA(c, cudaSetDevice(c->device));
  const size_t n = has_key_tables(c) ? c->n_keys : 0;
  if (n_slots != n) return fail_args(c, entry, ("n_slots is " + std::to_string(n_slots) + ", hs_key_slots is " + std::to_string(n)).c_str());
  if (expect_pks && n && !c->explicit_committee) return fail_args(c, entry, "key-cache tables are audited with expect_pks == NULL");
  HS_TRY(audit_stream(c));
  std::vector<uint8_t> live(n, 1);  // a staged slot is not in service
  if (c->explicit_committee)
    std::transform(c->h_key_live.begin(), c->h_key_live.begin() + n, live.begin(), [](uint8_t v) { return v == SLOT_STAGED ? 0 : v; });
  r = audit_run{};
  r.n_slots = n;
  if (windows) r.size_windows(c->cp, n);
  const size_t res_bytes = 8 + 4 * (2 + n + r.win_words);
  h2d_stage in;
  const size_t s_res = in.add(nullptr, res_bytes), s_pks = in.add(expect_pks, expect_pks ? n * 32 : 0),
               s_live = in.add(expect_live, expect_live ? 4 * ((n + 31) / 32) : 0), s_mirror = in.add(live.data(), n),
               s_ok = in.add(nullptr, n);
  HS_TRY(in.upload(c, A.scratch, A.stream));
  uint8_t *res = in.ptr(s_res);
  HS_CUDA(c, cudaMemsetAsync(res, 0xff, 8, A.stream));
  HS_CUDA(c, cudaMemsetAsync(res + 8, 0, res_bytes - 8, A.stream));
  const audit_out O{reinterpret_cast<unsigned long long *>(res), reinterpret_cast<uint32_t *>(res + 8)};
  uint32_t *const wbits = reinterpret_cast<uint32_t *>(res + 8) + 2 + n;
  const audit_wins key_wins{wbits, 0}, base_wins{wbits + r.base_word, 0};
  const auto kw = [&](size_t b) { return audit_wins{wbits, b * (size_t)(c->cp.na + 1)}; };
  if (n) {
    HS_TRY(launch_slot_audit(c, A.stream, ctx_tables(c).T, c->keys.key_flags, in.ptr(s_mirror), expect_pks ? in.ptr(s_pks) : nullptr,
                             expect_live ? reinterpret_cast<const uint32_t *>(in.ptr(s_live)) : nullptr, in.ptr(s_ok), O));
    if (!slice)
      HS_TRY(launch_table_audit(c, A.stream, c->keys.atables, nullptr, n, c->a_table_entries, c->cp.wa, c->cp.na, c->keys.pks, in.ptr(s_ok), O,
                                nullptr, windows ? &key_wins : nullptr));
    for (const auto &[b, e] : slice ? slice->tables : std::vector<std::pair<size_t, size_t>>{})  // a run: the same form on that window of the arrays
      if (b < e && e <= n) {
        const audit_wins w = kw(b);
        HS_TRY(launch_table_audit(c, A.stream, c->keys.atables + b * c->a_table_entries, nullptr, e - b, c->a_table_entries, c->cp.wa, c->cp.na,
                                  c->keys.pks + 32 * b, in.ptr(s_ok) + b, audit_out{O.first, O.bits + b}, nullptr, windows ? &w : nullptr));
      }
  }
  if (!slice) {
    HS_TRY(launch_table_audit(c, A.stream, c->d_btable, nullptr, 1, comb_table_entries(c->cp.wb), c->cp.wb, c->cp.nb, nullptr, nullptr, O,
                              nullptr, windows ? &base_wins : nullptr));
  } else if (slice->base_count) {
    const base_range R{slice->base_first, slice->base_count};
    HS_TRY(launch_table_audit(c, A.stream, c->d_btable, nullptr, 1, comb_table_entries(c->cp.wb), c->cp.wb, c->cp.nb, nullptr, nullptr, O, &R,
                              windows ? &base_wins : nullptr));
  }
  HS_CUDA(c, cudaEventRecord(A.done, A.stream));
  r.gen = c->key_gen;
  r.d_res = res;
  r.res.resize(res_bytes);
  return HS_OK;
}
// Without c->mu: waits for the kernels and reads the findings back.  HS_ERR_ARG (`changed`) when the key tables changed meanwhile.
static int audit_collect(hs_ctx *c, const char *entry, const char *changed, audit_run &r) {
  audit_state &A = c->audit;
  HS_CUDA(c, cudaEventSynchronize(A.done));
  HS_CUDA(c, cudaMemcpyAsync(r.res.data(), r.d_res, r.res.size(), cudaMemcpyDeviceToHost, A.stream));
  HS_CUDA(c, cudaStreamSynchronize(A.stream));
  std::lock_guard<std::mutex> g(c->mu);
  if (c->key_gen != r.gen) return fail_args(c, entry, changed);
  return HS_OK;
}

extern "C" int hs_table_audit(hs_ctx *c, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots, uint8_t *out_slot_bits,
                              uint32_t *out_failed) {
  if (!c || !out_failed) return fail(c, HS_ERR_ARG, "hs_table_audit: bad argument");
  std::lock_guard<std::mutex> ga(c->audit_mu);
  audit_run r;
  {
    std::lock_guard<std::mutex> g(c->mu);
    HS_TRY(audit_enqueue_locked(c, "hs_table_audit", expect_pks, expect_live, n_slots, r));
  }
  HS_TRY(audit_collect(c, "hs_table_audit", "key tables changed during the audit; run it again", r));
  const uint32_t failed = r.failed();
  for (size_t s = 0; s < n_slots && out_slot_bits; s++) out_slot_bits[s] = (uint8_t)r.bits()[2 + s];
  *out_failed = failed;
  return failed ? fail(c, HS_ERR_SELFTEST, audit_message(r.first(), n_slots, r.bits()).c_str()) : HS_OK;
}

// ---- building and proving a list of key slots off the verify path (hs_table_repair, hs_committee_stage)
// The comb tables of `slots` (their key bytes already in keys.pks), built on the audit's stream by one k_build_comb launch, with the
// flag bytes into the audit's scratch, then proved by one k_table_audit launch against those key bytes; a key that does not decompress
// has no table to prove.  Enqueued under c->mu by slot_build_enqueue, waited for and read back without it by slot_build_collect.  The
// caller holds audit_mu, so the audit's stream, event and scratch are its own.
struct slot_build {
  size_t n = 0;
  const uint8_t *d_out = nullptr;  // flag bytes (n), then at res_off an audit_out: first (8 bytes), bits[2 + n]
  size_t res_off = 0;
  std::vector<uint8_t> h;          // d_out read back
  uint8_t flag(size_t k) const { return h[k]; }
  bool proved(size_t k) const {    // the table of list position k passed, or the key has none
    uint32_t bits;
    memcpy(&bits, h.data() + res_off + 8 + 4 * (2 + k), 4);
    return !(h[k] & 1u) || !bits;
  }
};
static int slot_build_enqueue(hs_ctx *c, const std::vector<uint32_t> &slots, slot_build &B) {
  audit_state &A = c->audit;
  const size_t n = slots.size();
  HS_TRY(audit_stream(c));
  h2d_stage st;
  const size_t s_slots = st.add(slots.data(), 4 * n), s_flags = st.add(nullptr, n), s_res = st.add(nullptr, 8 + 4 * (2 + n));
  HS_TRY(st.upload(c, A.scratch, A.stream));
  uint8_t *out = st.ptr(s_flags), *res = st.ptr(s_res);
  HS_CUDA(c, cudaMemsetAsync(out, 0, st.total - st.sec[s_flags].off, A.stream));
  HS_CUDA(c, cudaMemsetAsync(res, 0xff, 8, A.stream));
  const uint32_t *d_slots = reinterpret_cast<const uint32_t *>(st.ptr(s_slots));
  HS_TRY(launch_build(c, c->keys.pks, d_slots, n, 1, c->cp.wa, c->cp.na, c->keys.atables, out, A.stream));
  HS_TRY(launch_table_audit(c, A.stream, c->keys.atables, d_slots, n, c->a_table_entries, c->cp.wa, c->cp.na, c->keys.pks, out,
                            audit_out{reinterpret_cast<unsigned long long *>(res), reinterpret_cast<uint32_t *>(res + 8)}));
  HS_CUDA(c, cudaEventRecord(A.done, A.stream));  // the key-cache paths, registration and updates wait for it before they rewrite
  B.n = n;
  B.d_out = out;
  B.res_off = (size_t)(res - out);
  B.h.resize(st.total - st.sec[s_flags].off);
  return HS_OK;
}
static cudaError_t slot_build_collect(hs_ctx *c, slot_build &B) {
  audit_state &A = c->audit;
  cudaError_t e = cudaEventSynchronize(A.done);
  if (e == cudaSuccess) e = cudaMemcpyAsync(B.h.data(), B.d_out, B.h.size(), cudaMemcpyDeviceToHost, A.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(A.stream);
  return e;
}

// ---- repair of what the audit finds (hs_table_repair)
// Empties the signature cache and the certificate cache of every verify queue of the context (under c->mu, the device drained): a
// record accepted against a wrong table must not be answered from a cache.  Requests in flight complete as they would.
static int flush_queue_caches(hs_ctx *c) {
  std::lock_guard<std::mutex> gq(c->queues_mu);
  for (hs_queue *q : c->queues) {
    if (q->d_sig) HS_TRY(sig_cache_set_locked(q, q->sig_bmask + 1));
    std::lock_guard<std::mutex> g(q->mu);
    cert_evict_locked(q, 0);
  }
  return HS_OK;
}

// Repairs the findings of audit `first` from the authority (the caller's map, else the host mirror), under the lock `g` of c->mu.
// The base-point table is rebuilt in place with the device drained.  Slots with a KEY, FLAG or TABLE finding that the authority holds
// dead are taken out of service as a removal would; the others (R) are rebuilt.  A committee's R is taken out of service (flag 0,
// SLOT_REPAIR: out of the hash table), rebuilt and proven on the audit's stream without the mutex, and each slot whose table passes
// goes back.  The key cache's R is rebuilt with the mutex held throughout: a learned key taken out of the hash table would be learned
// again.  HS_ERR_ARG `changed` when the key tables changed during the repair; what the repair took out of service is put back first.
static int repair_locked(hs_ctx *c, std::unique_lock<std::mutex> &g, const audit_run &first, const uint8_t *expect_pks,
                         const uint32_t *expect_live, const char *changed) {
  audit_state &A = c->audit;
  if (c->key_gen != first.gen) return fail_args(c, "hs_table_repair", changed);
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaDeviceSynchronize());  // nothing that read a wrong table is in flight, verify queue launches included
  const bool committee = c->explicit_committee;
  const uint32_t *bits = first.bits();
  if (bits[0]) {
    HS_TRY(launch_build(c, nullptr, nullptr, 1, 0, c->cp.wb, c->cp.nb, c->d_btable, nullptr, c->stream));
    HS_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  std::vector<uint32_t> R;
  for (size_t s = 0; s < first.n_slots; s++) {
    if (!(bits[2 + s] & (HS_AUDIT_KEY | HS_AUDIT_FLAG | HS_AUDIT_TABLE))) continue;
    // A staged slot stays staged with flag 0: its commit writes its proved flag byte.
    const bool staged = committee && c->h_key_live[s] == SLOT_STAGED;
    const bool live = !staged && (!committee || (expect_live ? (expect_live[s >> 5] >> (s & 31)) & 1u : (expect_pks || c->h_key_live[s])));
    if (live) {
      R.push_back((uint32_t)s);
      if (expect_pks) memcpy(c->h_pks.data() + 32 * s, expect_pks + 32 * s, 32);
    }
    if (committee && !staged) c->h_key_live[s] = live ? SLOT_REPAIR : 0;
    HS_CUDA(c, cudaMemsetAsync(c->keys.key_flags + s, 0, 1, c->stream));
  }
  if (first.n_slots) HS_TRY(publish_hash(c));  // also the whole repair of a LOOKUP finding
  HS_CUDA(c, cudaStreamSynchronize(c->stream));
  HS_TRY(flush_queue_caches(c));
  const uint64_t gen = ++c->key_gen;
  if (R.empty()) return HS_OK;
  // Rebuild R on the audit's stream: key bytes, then every table in one build launch and one proof launch.
  for (uint32_t s : R) HS_CUDA(c, cudaMemcpyAsync(c->keys.pks + 32 * (size_t)s, c->h_pks.data() + 32 * (size_t)s, 32, cudaMemcpyHostToDevice, A.stream));
  slot_build B;
  HS_TRY(slot_build_enqueue(c, R, B));
  if (committee) g.unlock();
  const cudaError_t e = slot_build_collect(c, B);
  if (committee) g.lock();
  if (e != cudaSuccess) return fail(c, HS_ERR_CUDA, "hs_table_repair: rebuild", e);  // R stays out of service
  // Back into service: each slot of R an update or a registration did not take over meanwhile, whose table passed (a key that does
  // not decompress has none to prove).  A slot whose table failed stays out of service, and the final audit reports it.
  for (size_t k = 0; k < R.size(); k++) {
    const size_t s = R[k];
    if (committee && (!c->explicit_committee || s >= c->n_keys || c->h_key_live[s] != SLOT_REPAIR)) continue;
    if (!B.proved(k)) continue;
    HS_CUDA(c, cudaMemcpyAsync(c->keys.key_flags + s, B.h.data() + k, 1, cudaMemcpyHostToDevice, c->stream));
    if (committee) c->h_key_live[s] = SLOT_LIVE;
  }
  if (committee && c->explicit_committee) HS_TRY(publish_hash(c));
  HS_CUDA(c, cudaStreamSynchronize(c->stream));
  const bool same = c->key_gen == gen;
  c->key_gen++;
  return same ? HS_OK : fail_args(c, "hs_table_repair", changed);
}

extern "C" int hs_table_repair(hs_ctx *c, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots, uint8_t *out_slot_bits,
                               uint32_t *out_found, uint32_t *out_failed) {
  if (!c || !out_found || !out_failed) return fail(c, HS_ERR_ARG, "hs_table_repair: bad argument");
  const char *changed = "key tables changed during the repair; run it again";
  std::lock_guard<std::mutex> ga(c->audit_mu);
  audit_run first, last;
  {
    std::lock_guard<std::mutex> g(c->mu);
    HS_TRY(audit_enqueue_locked(c, "hs_table_repair", expect_pks, expect_live, n_slots, first));
  }
  HS_TRY(audit_collect(c, "hs_table_repair", changed, first));
  const uint32_t found = first.failed();
  if (found) {
    {
      std::unique_lock<std::mutex> g(c->mu);
      HS_TRY(repair_locked(c, g, first, expect_pks, expect_live, changed));
      HS_TRY(audit_enqueue_locked(c, "hs_table_repair", expect_pks, expect_live, n_slots, last));
    }
    HS_TRY(audit_collect(c, "hs_table_repair", changed, last));
  }
  const uint32_t failed = found ? last.failed() : 0u;
  for (size_t s = 0; s < n_slots && out_slot_bits; s++) out_slot_bits[s] = (uint8_t)first.bits()[2 + s];
  *out_found = found;
  *out_failed = failed;
  return failed ? fail(c, HS_ERR_SELFTEST, audit_message(last.first(), n_slots, last.bits()).c_str()) : HS_OK;
}

// ---- mend of what the audit finds, in place and with no drain (hs_table_mend, and the scrub with hs_scrub_mend)
// What the mend takes of audit r (run with its window findings): every flagged window of the base-point table, whose anchor B is a
// constant; and the flagged windows of each slot whose only finding is TABLE, unless its anchor failed with no map (have_map) to
// confirm its key bytes: bytes that changed but still decompress look exactly like a bad anchor, and a table rebuilt from them would
// hold the wrong key's multiples.  Everything else is left to hs_table_repair.
struct mend_plan {
  std::vector<mend_item> base, keys;  // the windows to recompute
  std::vector<uint32_t> slots;        // the slots of `keys`, in slot order
  uint32_t left = 0;                  // the HS_AUDIT_* classes left
  uint64_t windows_left = 0, slots_left = 0;
};
static mend_plan mend_plan_of(const audit_run &r, bool have_map) {
  mend_plan P;
  const uint32_t *bits = r.bits();
  if (bits[0]) {
    for (int i = 0; i < r.nb; i++)
      if (r.base_win(i)) P.base.push_back({HS_MEND_BASE, (uint32_t)i});
    if (P.base.empty()) P.left |= HS_AUDIT_BASE;
  }
  P.left |= bits[1];
  for (size_t s = 0; s < r.n_slots; s++) {
    if (!bits[2 + s]) continue;
    const size_t before = P.keys.size();
    if (bits[2 + s] == HS_AUDIT_TABLE && (have_map || !r.key_win(s, r.na)))
      for (int i = 0; i < r.na; i++)
        if (r.key_win(s, i)) P.keys.push_back({(uint32_t)s, (uint32_t)i});
    if (P.keys.size() > before) {
      P.slots.push_back((uint32_t)s);
      continue;
    }
    P.left |= bits[2 + s];
    P.slots_left++;
    for (int i = 0; i < r.na; i++) P.windows_left += r.key_win(s, i) ? 1 : 0;
  }
  return P;
}
// Threads of one k_mend_windows launch: a wave of the device at 256 threads per SM, so its staging (6,240 bytes a thread: 211 MB on
// 132 SMs) stays bounded whatever the window; a 24-bit base window (2^23 entries, 131,072 threads) takes four launches.
static size_t mend_chunk(const hs_ctx *c) { return (size_t)c->n_sms * 256; }
// One mend of plan P: enqueued under c->mu by mend_enqueue_locked, waited for and read back without it by mend_collect.  The proof
// audits each mended window again: the base-point table's by the range form over the window and the next (whose entry 1 links to
// it), the slots' by the listed form over their whole tables.  The caller holds audit_mu.
struct mend_run {
  const uint8_t *d_out = nullptr;  // entries rewritten (8 bytes), then the proof's results
  std::vector<uint8_t> h;
  audit_run proof;                 // its slot t is P.slots[t]
  uint64_t rewritten() const {
    uint64_t v;
    memcpy(&v, h.data(), 8);
    return v;
  }
};
static int mend_enqueue_locked(hs_ctx *c, const char *entry, const char *changed, const audit_run &first, const mend_plan &P, mend_run &M) {
  audit_state &A = c->audit;
  // The last check before the stores: a registration, update, commit or key-cache change since the audit leaves nothing stored.  Any
  // later one waits for A.done (audit_fence, or a drained device) before it writes, so it lands after these stores.
  if (c->key_gen != first.gen) return fail_args(c, entry, changed);
  HS_CUDA(c, cudaSetDevice(c->device));
  const size_t k = P.slots.size();
  M.proof.n_slots = k;
  M.proof.size_windows(c->cp, k);
  const size_t proof_bytes = 8 + 4 * (2 + k + M.proof.win_words);
  std::vector<mend_item> items(P.base);
  items.insert(items.end(), P.keys.begin(), P.keys.end());
  const std::vector<uint8_t> ones(k, 1);
  h2d_stage st;
  const size_t s_items = st.add(items.data(), items.size() * sizeof(mend_item)), s_slots = st.add(P.slots.data(), 4 * k),
               s_ok = st.add(ones.data(), k), s_out = st.add(nullptr, 8 + proof_bytes);
  HS_TRY(st.upload(c, A.scratch, A.stream));
  uint8_t *out = st.ptr(s_out), *res = out + 8;
  HS_CUDA(c, cudaMemsetAsync(out, 0, 8 + proof_bytes, A.stream));
  HS_CUDA(c, cudaMemsetAsync(res, 0xff, 8, A.stream));
  unsigned long long *rewritten = reinterpret_cast<unsigned long long *>(out);
  const mend_item *d_items = reinterpret_cast<const mend_item *>(st.ptr(s_items));
  const size_t chunk = mend_chunk(c);
  const auto mend = [&](const mend_item *its, size_t n_items, int W, ge_niels *tables, size_t table_entries, const uint8_t *pks) -> int {
    const uint64_t total = (uint64_t)n_items * (((uint64_t)1 << (W - 1)) / HS_BUILD_BLOCK);
    for (uint64_t b = 0; b < total; b += chunk) {
      const uint64_t nb = std::min<uint64_t>(chunk, total - b);
      k_mend_windows<<<blocks_for(nb), HS_THREADS, 0, A.stream>>>(its, b, nb, W, tables, table_entries, pks,
                                                                  static_cast<ge_niels *>(A.stage.p.get()), rewritten);
      c->launches++;
      HS_CUDA(c, cudaGetLastError());
    }
    return HS_OK;
  };
  if (!P.base.empty()) HS_TRY(mend(d_items, P.base.size(), c->cp.wb, c->d_btable, 0, nullptr));
  if (k) HS_TRY(mend(d_items + P.base.size(), P.keys.size(), c->cp.wa, c->keys.atables, c->a_table_entries, c->keys.pks));
  const audit_out O{reinterpret_cast<unsigned long long *>(res), reinterpret_cast<uint32_t *>(res + 8)};
  uint32_t *const wbits = reinterpret_cast<uint32_t *>(res + 8) + 2 + k;
  const uint64_t E = comb_table_entries(c->cp.wb), stride = comb_window_stride(c->cp.wb);
  const audit_wins base_wins{wbits + M.proof.base_word, 0}, key_wins{wbits, 0};
  for (size_t j = 0; j < P.base.size();) {  // runs of consecutive windows, each with the window after it
    size_t e = j + 1;
    while (e < P.base.size() && P.base[e].win == P.base[e - 1].win + 1) e++;
    const uint64_t from = P.base[j].win * stride;
    const base_range R{from, std::min<uint64_t>(E, (P.base[e - 1].win + 2) * stride) - from};
    HS_TRY(launch_table_audit(c, A.stream, c->d_btable, nullptr, 1, E, c->cp.wb, c->cp.nb, nullptr, nullptr, O, &R, &base_wins));
    j = e;
  }
  if (k)
    HS_TRY(launch_table_audit(c, A.stream, c->keys.atables, reinterpret_cast<const uint32_t *>(st.ptr(s_slots)), k, c->a_table_entries, c->cp.wa,
                              c->cp.na, c->keys.pks, st.ptr(s_ok), O, nullptr, &key_wins));
  HS_CUDA(c, cudaEventRecord(A.done, A.stream));  // registration, updates and the key-cache paths wait for it before they rewrite
  M.d_out = out;
  M.h.resize(8 + proof_bytes);
  return HS_OK;
}
static int mend_collect(hs_ctx *c, mend_run &M) {
  audit_state &A = c->audit;
  HS_CUDA(c, cudaEventSynchronize(A.done));
  HS_CUDA(c, cudaMemcpyAsync(M.h.data(), M.d_out, M.h.size(), cudaMemcpyDeviceToHost, A.stream));
  HS_CUDA(c, cudaStreamSynchronize(A.stream));
  M.proof.res.assign(M.h.begin() + 8, M.h.end());
  return HS_OK;
}
// Mends what audit `first` found (run with its window findings) and proves it; *left: the classes left (not mendable, or still failing
// the proof).  Never drains the device and never changes a slot's service state: the context's mutex is held to enqueue and, when an
// entry was rewritten, to empty every verify queue's caches as a repair does (a record may have been decided against the wrong entry).
// The caller holds audit_mu.
static int mend_found(hs_ctx *c, const char *entry, const char *changed, const audit_run &first, bool have_map, uint32_t &left) {
  c->mend_stats[MEND_CALLS]++;
  const mend_plan P = mend_plan_of(first, have_map);
  left = P.left;
  uint64_t windows_left = P.windows_left, slots_left = P.slots_left;
  const size_t windows = P.base.size() + P.keys.size();
  if (windows) {
    const uint64_t threads = std::max<uint64_t>(P.base.empty() ? 0 : ((uint64_t)1 << (c->cp.wb - 1)) / HS_BUILD_BLOCK,
                                                P.keys.empty() ? 0 : ((uint64_t)1 << (c->cp.wa - 1)) / HS_BUILD_BLOCK);
    HS_TRY(ensure(c, c->audit.stage, std::min<uint64_t>(mend_chunk(c), threads * windows) * (HS_BUILD_BLOCK + 1) * sizeof(ge_niels)));
    mend_run M;
    {
      std::lock_guard<std::mutex> g(c->mu);
      HS_TRY(mend_enqueue_locked(c, entry, changed, first, P, M));
    }
    HS_TRY(mend_collect(c, M));
    const audit_run &pr = M.proof;
    if (pr.bits()[0]) {
      left |= HS_AUDIT_BASE;
      for (int i = 0; i < pr.nb; i++) windows_left += pr.base_win(i) ? 1 : 0;
    }
    for (size_t t = 0; t < pr.n_slots; t++) {
      if (!pr.bits()[2 + t]) continue;
      left |= pr.bits()[2 + t];
      slots_left++;
      for (int i = 0; i < pr.na; i++) windows_left += pr.key_win(t, i) ? 1 : 0;
    }
    const uint64_t rewritten = M.rewritten();
    c->mend_stats[MEND_WINDOWS] += windows;
    c->mend_stats[MEND_REWRITTEN] += rewritten;
    if (rewritten) {
      std::lock_guard<std::mutex> g(c->mu);
      HS_TRY(flush_queue_caches(c));
      c->mend_stats[MEND_FLUSHES]++;
    }
  }
  c->mend_stats[MEND_WINDOWS_LEFT] += windows_left;
  c->mend_stats[MEND_SLOTS_LEFT] += slots_left;
  return HS_OK;
}

extern "C" int hs_table_mend(hs_ctx *c, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots, uint8_t *out_slot_bits,
                             uint32_t *out_found, uint32_t *out_left) {
  if (!c || !out_found || !out_left) return fail(c, HS_ERR_ARG, "hs_table_mend: bad argument");
  const char *entry = "hs_table_mend", *changed = "key tables changed during the mend; run it again";
  std::lock_guard<std::mutex> ga(c->audit_mu);
  audit_run first;
  {
    std::lock_guard<std::mutex> g(c->mu);
    HS_TRY(audit_enqueue_locked(c, entry, expect_pks, expect_live, n_slots, first, nullptr, true));
  }
  HS_TRY(audit_collect(c, entry, changed, first));
  uint32_t left = 0;
  HS_TRY(mend_found(c, entry, changed, first, expect_pks != nullptr, left));
  for (size_t s = 0; s < n_slots && out_slot_bits; s++) out_slot_bits[s] = (uint8_t)first.bits()[2 + s];
  *out_found = first.failed();
  *out_left = left;
  if (!left) return HS_OK;
  return fail(c, HS_ERR_SELFTEST, ("hs_table_mend: findings of HS_AUDIT_* classes " + std::to_string(left) + " left to hs_table_repair").c_str());
}

extern "C" int hs_table_mend_stats(hs_ctx *c, uint64_t out[HS_MEND_STATS]) {
  if (!c || !out) return HS_ERR_ARG;
  for (int k = 0; k < MEND_NSTATS; k++) out[k] = c->mend_stats[k].load();
  return HS_OK;
}

// ---- staged committee change (hs_committee_stage / hs_committee_commit / hs_committee_discard)
// stage(A, R) + commit leaves the context as hs_committee_update(A, none) + hs_committee_update(none, R) would.  The stage picks the
// slots as update does and marks them SLOT_STAGED (out of service: not in the hash table, flag 0), then builds and proves their tables
// off the verify path as a repair does.  The commit writes the proved flags, takes R out of service and publishes the hash table.
extern "C" int hs_committee_stage(hs_ctx *c, const uint8_t *add_pks, size_t n_add, const uint32_t *remove_idx, size_t n_remove,
                                  uint32_t *out_add_idx) {
  const char *entry = "hs_committee_stage";
  if (!c || (n_add && (!add_pks || !out_add_idx)) || (n_remove && !remove_idx)) return fail_args(c, entry, "bad argument");
  std::lock_guard<std::mutex> ga(c->audit_mu);
  slot_plan P;
  slot_build B;
  uint64_t gen = 0;
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (!committee_registered(c)) return fail_args(c, entry, "no committee registered");
    if (c->stage.busy) return fail_args(c, entry, "a stage is already pending (commit or discard it)");
    plan_adds(c, add_pks, n_add, SLOT_STAGED, P);
    if (P.full) return fail(c, HS_ERR_NOMEM, "hs_committee_stage: too few free and spare slots (use hs_committee_update)");
    for (size_t i = 0; i < n_remove; i++)  // against the slots in use once the additions are in, as the second update would check
      if (remove_idx[i] >= P.live.size()) return fail_args(c, entry, "remove index out of range");
    HS_CUDA(c, cudaSetDevice(c->device));
    committee_stage &S = c->stage;
    S.busy = true;
    S.fresh = P.fresh;
    S.remove.assign(remove_idx, remove_idx + n_remove);
    for (uint32_t s : P.fresh) S.keys.insert(S.keys.end(), P.pks.begin() + 32 * (size_t)s, P.pks.begin() + 32 * (size_t)s + 32);
    c->h_key_live = P.live;
    gen = c->key_gen;
    // Key bytes of slots out of service: no launch resolves a key to them, and a committee-indexed record naming one rejects on its flag.
    const auto enqueue = [&]() -> int {
      if (P.fresh.empty()) return HS_OK;
      HS_TRY(audit_stream(c));
      for (size_t k = 0; k < P.fresh.size(); k++)
        HS_CUDA(c, cudaMemcpyAsync(c->keys.pks + 32 * (size_t)P.fresh[k], S.keys.data() + 32 * k, 32, cudaMemcpyHostToDevice, c->audit.stream));
      return slot_build_enqueue(c, P.fresh, B);
    };
    if (const int rc = enqueue()) {
      stage_drop(c);
      return rc;
    }
  }
  const cudaError_t e = P.fresh.empty() ? cudaSuccess : slot_build_collect(c, B);
  std::lock_guard<std::mutex> g(c->mu);
  if (c->key_gen != gen) return fail_args(c, entry, "a registration or update ran during the stage; stage again");  // it dropped the stage
  if (e != cudaSuccess) {
    stage_drop(c);
    return fail(c, HS_ERR_CUDA, "hs_committee_stage: build", e);
  }
  for (size_t k = 0; k < P.fresh.size(); k++)
    if (!B.proved(k)) {
      stage_drop(c);
      return fail(c, HS_ERR_SELFTEST, ("hs_committee_stage: slot " + std::to_string(P.fresh[k]) + ": the staged comb table failed its proof (TABLE)").c_str());
    }
  c->stage.flags.assign(B.h.begin(), B.h.begin() + P.fresh.size());
  c->stage.ready = true;
  std::copy(P.idx.begin(), P.idx.end(), out_add_idx);
  return HS_OK;
}

// The commit of a staged registration, under both mutexes: drains the device as registration does, releases the key cache's state and
// moves the proved store in.  The replaced store goes to `old`, which the caller frees once it has released the mutexes.
static int register_commit_locked(hs_ctx *c, key_store &old) {
  HS_CUDA(c, cudaSetDevice(c->device));
  // A queue enqueues a launch only while it holds c->mu, so nothing launched against the old indices survives this line.
  HS_CUDA(c, cudaDeviceSynchronize());
  committee_stage S = std::move(c->stage);
  old = std::move(c->keys);
  cache_release(c);  // bumps key_gen and map_gen: the scrub pauses, and an audit against the old map is refused
  c->learn_pending = false;
  c->cache_full = false;
  c->cache_enabled = c->cache_wanted;
  c->keys = std::move(S.store);
  set_window(c->cp, true, S.wa);
  c->a_table_entries = comb_table_entries(S.wa);
  c->n_keys = S.keys.size() / 32;
  c->key_capacity = S.capacity;
  c->explicit_committee = true;
  c->h_pks = std::move(S.keys);
  c->h_index = std::move(S.index);
  c->h_key_live.assign(c->n_keys, SLOT_LIVE);
  return HS_OK;
}

extern "C" int hs_committee_commit(hs_ctx *c) {
  if (!c) return HS_ERR_ARG;
  key_store old;  // declared before the locks: freed after both are released (cudaFree of the old tables waits for the device)
  std::lock_guard<std::mutex> ga(c->audit_mu);  // before mu: the commit never waits for an audit while it holds the mutex
  std::lock_guard<std::mutex> g(c->mu);
  committee_stage &S = c->stage;
  if (S.ready && S.whole) return register_commit_locked(c, old);
  if (!S.ready || !committee_registered(c))
    return fail_args(c, "hs_committee_commit", "no stage pending (none was made, or a registration or update discarded it)");
  HS_CUDA(c, cudaSetDevice(c->device));
  // A launch in flight that resolved a key to a removed slot must not see its flag cleared.  Adding slots disturbs no launch in flight.
  if (!S.remove.empty()) HS_CUDA(c, cudaDeviceSynchronize());
  c->key_gen++;
  c->map_gen++;
  for (size_t k = 0; k < S.fresh.size(); k++) {
    const uint32_t s = S.fresh[k];
    if (s >= c->n_keys) {  // a spare: the spares a stage takes follow n_keys without a gap
      c->n_keys = (size_t)s + 1;
      c->h_pks.resize(c->n_keys * 32);
    }
    memcpy(c->h_pks.data() + 32 * (size_t)s, S.keys.data() + 32 * k, 32);
    c->h_key_live[s] = SLOT_LIVE;
    HS_CUDA(c, cudaMemcpyAsync(c->keys.key_flags + s, S.flags.data() + k, 1, cudaMemcpyHostToDevice, c->stream));
  }
  for (uint32_t s : S.remove) {
    c->h_key_live[s] = 0;
    HS_CUDA(c, cudaMemsetAsync(c->keys.key_flags + s, 0, 1, c->stream));
  }
  stage_drop(c);
  return publish_hash(c);  // behind the flag bytes on the same stream; the key bytes were in place when the stage returned
}

extern "C" int hs_committee_discard(hs_ctx *c) {
  if (!c) return HS_ERR_ARG;
  key_store staged;  // a staged registration's store, freed after both locks are released
  std::lock_guard<std::mutex> ga(c->audit_mu);
  std::lock_guard<std::mutex> g(c->mu);
  staged = std::move(c->stage.store);
  stage_drop(c);
  return HS_OK;
}

// ---- staged registration (hs_committee_stage_register; hs_committee_commit and hs_committee_discard apply or drop it)
// Test builds XOR one armed byte of the staged store before its proof (hs_test_poke_staged); the product build does nothing.
static int staged_poke_apply(hs_ctx *c, key_store &K, size_t N, size_t entries, cudaStream_t stream);
// stage_register(P, w) + commit leaves the context as hs_committee_register(P) leaves one whose window came out as w.  Under c->mu the
// stage checks the arguments, picks the geometry and marks itself pending; then, holding only audit_mu, it builds a whole new key store
// beside the live one on the audit's stream and proves it with the audit's checks.  Nothing live is read or written until the commit.
extern "C" int hs_committee_stage_register(hs_ctx *c, const uint8_t *pks, size_t N, int key_bits, uint32_t *out_valid_bitmap,
                                           int *out_key_bits) {
  const char *entry = "hs_committee_stage_register";
  if (!c || !pks || N == 0 || N >= HS_NO_KEY || (key_bits && (key_bits < 8 || key_bits > 17))) return fail_args(c, entry, "bad argument");
  std::lock_guard<std::mutex> ga(c->audit_mu);
  const size_t capk = committee_capacity(N);
  int wa = 0;
  comb_params cp{};
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (c->stage.busy) return fail_args(c, entry, "a stage is already pending (commit or discard it)");
    if (key_bits && c->wa_forced && key_bits != c->wa_forced) return fail_args(c, entry, "key_bits differs from the context's forced window");
    HS_CUDA(c, cudaSetDevice(c->device));
    size_t budget = 0;  // with the live store still allocated
    HS_TRY(committee_budget(c, budget));
    const int want = key_bits ? key_bits : c->wa_forced;
    for (int w : {17, 16, 15, 14, 13, 12, 11, 10, 9, 8})
      if ((!want || w == want) && capk * comb_table_entries(w) * sizeof(ge_niels) <= budget) {
        wa = w;
        break;
      }
    if (!wa) return fail(c, HS_ERR_NOMEM, "hs_committee_stage_register: the tables do not fit in the table budget beside the live store");
    if (sc_ndigits_rt(wa) + c->cp.nb > HS_MAX_DIGITS) return fail_args(c, entry, "window combination exceeds HS_MAX_DIGITS");
    cp = c->cp;
    set_window(cp, true, wa);
    c->stage.busy = true;
    c->stage.whole = true;
  }
  key_index index;
  index.reset(capk);
  index.build(pks, N, [](size_t) { return true; });
  const size_t entries = comb_table_entries(wa);
  key_store K;
  std::vector<uint8_t> fl(N), res(8 + 4 * (2 + N));
  audit_state &A = c->audit;
  const int rc = [&]() -> int {
    HS_TRY(audit_stream(c));
    const cudaError_t e = make_key_store(K, capk, index.slots.size(), wa, A.stream);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(c, HS_ERR_NOMEM, "hs_committee_stage_register: the staged tables do not fit in device memory", e);
    }
    HS_CUDA(c, cudaMemcpyAsync(K.pks, pks, N * 32, cudaMemcpyHostToDevice, A.stream));
    HS_CUDA(c, cudaMemcpyAsync(K.slots, index.slots.data(), index.slots.size() * 4, cudaMemcpyHostToDevice, A.stream));
    HS_TRY(launch_build(c, K.pks, nullptr, N, 1, wa, cp.na, K.atables, K.key_flags, A.stream));
    HS_TRY(staged_poke_apply(c, K, N, entries, A.stream));  // test builds: hs_test_poke_staged; a no-op otherwise
    // The proof: every slot in service, its key bytes against the caller's, its flag byte and lookup, every hash entry, every table.
    const std::vector<uint8_t> live(N, SLOT_LIVE);
    h2d_stage in;
    const size_t s_res = in.add(nullptr, res.size()), s_pks = in.add(pks, N * 32), s_live = in.add(live.data(), N), s_ok = in.add(nullptr, N);
    HS_TRY(in.upload(c, A.scratch, A.stream));
    uint8_t *d_res = in.ptr(s_res);
    HS_CUDA(c, cudaMemsetAsync(d_res, 0xff, 8, A.stream));
    HS_CUDA(c, cudaMemsetAsync(d_res + 8, 0, res.size() - 8, A.stream));
    const audit_out O{reinterpret_cast<unsigned long long *>(d_res), reinterpret_cast<uint32_t *>(d_res + 8)};
    HS_TRY(launch_slot_audit(c, A.stream, store_tables(K, index, N, entries, cp).T, K.key_flags, in.ptr(s_live), in.ptr(s_pks), nullptr,
                             in.ptr(s_ok), O));
    HS_TRY(launch_table_audit(c, A.stream, K.atables, nullptr, N, entries, wa, cp.na, K.pks, in.ptr(s_ok), O));
    // No event: A.done orders the key-cache paths behind the audits, and learning need not wait for this build.
    HS_CUDA(c, cudaMemcpyAsync(res.data(), d_res, res.size(), cudaMemcpyDeviceToHost, A.stream));
    HS_CUDA(c, cudaMemcpyAsync(fl.data(), K.key_flags, N, cudaMemcpyDeviceToHost, A.stream));
    HS_CUDA(c, cudaStreamSynchronize(A.stream));
    const uint32_t *bits = reinterpret_cast<const uint32_t *>(res.data() + 8);
    uint32_t failed = bits[1];
    for (size_t s = 0; s < N; s++) failed |= bits[2 + s];
    if (failed) {
      uint64_t first;
      memcpy(&first, res.data(), 8);
      return fail(c, HS_ERR_SELFTEST, ("hs_committee_stage_register: the staged store failed its proof: " + audit_message(first, N, bits)).c_str());
    }
    return HS_OK;
  }();
  std::lock_guard<std::mutex> g(c->mu);
  committee_stage &S = c->stage;
  if (!S.busy || !S.whole) return fail_args(c, entry, "a registration or update ran during the stage; stage again");  // it dropped the stage
  if (rc != HS_OK) {
    S = {};
    return rc;
  }
  S.store = std::move(K);
  S.index = std::move(index);
  S.capacity = capk;
  S.wa = wa;
  S.keys.assign(pks, pks + N * 32);
  S.flags = fl;
  S.ready = true;
  if (out_valid_bitmap) {
    for (size_t w = 0; w < (N + 31) / 32; w++) out_valid_bitmap[w] = 0;
    for (size_t i = 0; i < N; i++)
      if (fl[i] & 1) out_valid_bitmap[i >> 5] |= 1u << (i & 31);
  }
  if (out_key_bits) *out_key_bits = wa;
  return HS_OK;
}

// ---- audit of a verify queue's signature cache (hs_queue_sig_audit, and the scrub's slices of it)
// The range an audit takes: buckets [first, first + n) (n = 0: none), and whether that is the whole table (a pass).
struct sig_audit_range {
  size_t first = 0, n = 0;
  bool pass = false;
};
// One k_sig_audit launch on the audit's stream: pick(buckets, sig_gen, range) chooses the range under c->mu from the table's size (0:
// the cache is off) and generation; false is HS_ERR_ARG.  Enqueued under c->mu, waited for and read back without it.  The caller holds
// audit_mu.  out: hs_queue_sig_audit's words; q's counters take the run.
template <class Pick>
static int sig_audit_run(hs_queue *q, const char *entry, Pick pick, uint64_t out[HS_QUEUE_SIG_AUDIT_OUT]) {
  hs_ctx *c = q->c;
  sig_audit_range r;
  {
    std::lock_guard<std::mutex> g(c->mu);  // the dispatcher and hs_queue_sig_cache change the table only under it
    if (!pick(q->d_sig ? q->sig_bmask + 1 : 0u, q->sig_gen, r))
      return fail_args(c, entry, "the signature cache is off, or the bucket range leaves its table");
    if (r.n) {
      HS_CUDA(c, cudaSetDevice(c->device));
      HS_TRY(audit_stream(c));
      if (!q->ev_audit) HS_CUDA(c, create(q->ev_audit));
      if (!q->d_audit) HS_CUDA(c, alloc(q->d_audit, 4 * sizeof(unsigned long long)));
      const cudaStream_t s = c->audit.stream;
      HS_CUDA(c, cudaMemsetAsync(q->d_audit, 0, 3 * sizeof(unsigned long long), s));
      HS_CUDA(c, cudaMemsetAsync(q->d_audit + 3, 0xff, sizeof(unsigned long long), s));
      HS_CUDA(c, launch_sig_audit(c, q->d_sig, (uint32_t)r.first, (uint32_t)r.n, q->d_audit, s));
      HS_CUDA(c, cudaEventRecord(q->ev_audit, s));  // sig_cache_set_locked waits for it before the table goes
    }
  }
  unsigned long long res[4] = {0, 0, 0, ~0ull};
  if (r.n) {
    HS_CUDA(c, cudaEventSynchronize(q->ev_audit));
    HS_CUDA(c, cudaMemcpyAsync(res, q->d_audit, sizeof(res), cudaMemcpyDeviceToHost, c->audit.stream));
    HS_CUDA(c, cudaStreamSynchronize(c->audit.stream));
  }
  const bool any = res[3] != ~0ull;
  const uint64_t v[HS_QUEUE_SIG_AUDIT_OUT] = {res[0], res[1], res[2], any ? res[3] >> 24 : UINT64_MAX, any ? (res[3] >> 16) & 0xff : 0,
                                              any ? (res[3] >> 8) & 0xff : 0, any ? res[3] & 0xff : 0};
  memcpy(out, v, sizeof(v));
  std::lock_guard<std::mutex> gq(q->mu);
  if (r.n) {
    q->astats[0]++;
    q->astats[1] += res[0];
    q->astats[2] += res[1];
    q->astats[3] += res[2];
  }
  if (r.pass) q->astats[4]++;
  return HS_OK;
}

extern "C" int hs_queue_sig_audit(hs_queue *q, size_t first_bucket, size_t n_buckets, uint64_t out[HS_QUEUE_SIG_AUDIT_OUT]) {
  if (!q || !out) return fail(q ? q->c : nullptr, HS_ERR_ARG, "hs_queue_sig_audit: bad argument");
  std::lock_guard<std::mutex> ga(q->c->audit_mu);
  return sig_audit_run(
      q, "hs_queue_sig_audit",
      [&](uint32_t buckets, uint32_t, sig_audit_range &r) {
        if (!buckets || first_bucket >= buckets || n_buckets > buckets - first_bucket) return false;
        r.first = first_bucket;
        r.n = n_buckets ? n_buckets : buckets - first_bucket;
        r.pass = r.first == 0 && r.n == buckets;
        return true;
      },
      out);
}

extern "C" int hs_queue_sig_audit_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_AUDIT_STATS]) {
  return queue_read_stats(q, "hs_queue_sig_audit_stats", out, &hs_queue::astats);
}

// ---- the engine-owned scrub of the live key tables (hs_scrub_start / hs_scrub_set_map / hs_scrub_stop / hs_scrub_stats)
// Takes the caller's map (or the engine's own) for the current slot map, under S.m: the rules of hs_table_audit.  A new map starts a
// new pass.
static int scrub_map_locked(hs_ctx *c, scrub_state &S, const char *entry, const uint8_t *pks, const uint32_t *live, size_t n_slots) {
  std::lock_guard<std::mutex> g(c->mu);
  const size_t n = has_key_tables(c) ? c->n_keys : 0;
  if (n_slots != n) return fail_args(c, entry, ("n_slots is " + std::to_string(n_slots) + ", hs_key_slots is " + std::to_string(n)).c_str());
  if (pks && n && !c->explicit_committee) return fail_args(c, entry, "key-cache tables are scrubbed with expect_pks == NULL");
  S.has_pks = pks && n;
  S.has_live = live && n;
  S.pks.assign(S.has_pks ? pks : nullptr, S.has_pks ? pks + 32 * n : nullptr);
  S.live.assign(S.has_live ? live : nullptr, S.has_live ? live + (n + 31) / 32 : nullptr);
  S.n_slots = n;
  S.map_gen = c->map_gen;
  S.next_slot = 0;
  S.next_base = 0;
  return HS_OK;
}
// What one tick found, for the callback: the classes found, those its proof still finds, the lowest slot with a finding.
struct scrub_report {
  uint32_t found = 0, failed = 0;
  size_t first_slot = SIZE_MAX;
};
// The runs of slots with a finding in `r` whose tables `sl` does not cover.
static std::vector<std::pair<size_t, size_t>> scrub_flagged_outside(const audit_run &r, const audit_slice &sl) {
  std::vector<std::pair<size_t, size_t>> out;
  for (size_t s = 0; s < r.n_slots; s++) {
    if (!r.bits()[2 + s] || std::any_of(sl.tables.begin(), sl.tables.end(), [s](const auto &t) { return t.first <= s && s < t.second; })) continue;
    if (!out.empty() && out.back().second == s) out.back().second = s + 1;
    else out.push_back({s, s + 1});
  }
  return out;
}
static uint64_t scrub_items(const audit_run &r) {  // the slots, the base-point table and the stray hash entries with a finding
  uint64_t k = (r.bits()[0] ? 1 : 0) + (r.bits()[1] ? 1 : 0);
  for (size_t s = 0; s < r.n_slots; s++) k += r.bits()[2 + s] ? 1 : 0;
  return k;
}
// One tick, under S.m: audit the next slice against the map; on a finding, audit the flagged slots' tables too, repair exactly what
// was found (repair_locked, as hs_table_repair does) and prove it by auditing the slice again.  A slot map newer than the scrub's map
// pauses the tick.  Errors other than a map change end the scrub.
static int scrub_tick(hs_ctx *c, scrub_state &S, scrub_report &rep) {
  const char *entry = "hs_scrub", *changed = "key tables changed during a scrub tick";
  const uint8_t *pks = S.has_pks ? S.pks.data() : nullptr;
  const uint32_t *live = S.has_live ? S.live.data() : nullptr;
  std::lock_guard<std::mutex> ga(c->audit_mu);
  audit_run r;
  audit_slice sl;
  uint64_t live_slots = 0;
  size_t s = S.next_slot;
  const uint64_t E = comb_table_entries(c->cp.wb);
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (c->map_gen != S.map_gen) {
      S.stats[SCRUB_PAUSED]++;
      return HS_OK;
    }
    // the next slots_per_tick slots in service, with the slots out of service up to the next one in service (they have no table)
    const auto in_service = [c](size_t k) { return !c->explicit_committee || (c->h_key_live[k] && c->h_key_live[k] != SLOT_STAGED); };
    while (s < S.n_slots && (live_slots < S.slots_per_tick || !in_service(s))) live_slots += in_service(s++) ? 1 : 0;
    sl.tables.push_back({S.next_slot, s});
    sl.base_first = S.next_base;
    sl.base_count = std::min<uint64_t>(S.base_per_tick, E - S.next_base);
    HS_TRY(audit_enqueue_locked(c, entry, pks, live, S.n_slots, r, &sl, S.mend));
  }
  int rc = audit_collect(c, entry, changed, r);
  if (rc == HS_ERR_ARG) {  // the slot map changed under the tick: nothing it found counts, and the next tick pauses
    S.stats[SCRUB_PAUSED]++;
    return HS_OK;
  }
  HS_TRY(rc);
  S.stats[SCRUB_TICKS]++;
  S.stats[SCRUB_SLOTS] += live_slots;
  S.stats[SCRUB_BASE] += sl.base_count;
  S.next_slot = s;
  S.next_base += sl.base_count;
  if (S.next_slot >= S.n_slots && S.next_base >= E) {
    S.stats[SCRUB_PASSES]++;
    S.next_slot = 0;
    S.next_base = 0;
  }
  if (!r.failed()) return HS_OK;
  // A slot the slot checks flagged outside the slice: its table decides what the repair rebuilds (key bytes that changed without a
  // map to compare them with show as LOOKUP here, and as TABLE through the anchor).
  const auto outside = scrub_flagged_outside(r, sl);
  if (!outside.empty()) {
    audit_run t;
    audit_slice st;
    st.tables = outside;
    {
      std::lock_guard<std::mutex> g(c->mu);
      HS_TRY(audit_enqueue_locked(c, entry, pks, live, S.n_slots, t, &st, S.mend));
    }
    rc = audit_collect(c, entry, changed, t);
    if (rc == HS_ERR_ARG) {
      S.stats[SCRUB_PAUSED]++;
      return HS_OK;
    }
    HS_TRY(rc);
    uint32_t *bits = reinterpret_cast<uint32_t *>(r.res.data() + 8);
    for (size_t k = 0; k < 2 + r.n_slots; k++) bits[k] |= t.bits()[k];
    for (size_t k = 0; k < r.win_words; k++) r.wins()[k] |= t.wins()[k];
    sl.tables.insert(sl.tables.end(), outside.begin(), outside.end());
  }
  rep.found = r.failed();
  for (size_t k = 0; k < r.n_slots && rep.first_slot == SIZE_MAX; k++)
    if (r.bits()[2 + k]) rep.first_slot = k;
  // With hs_scrub_mend, findings that can all be mended are mended (no drain, no slot out of service); anything else is repaired.
  const bool mend = S.mend && !mend_plan_of(r, pks != nullptr).left;
  uint32_t left = 0;
  if (mend) rc = mend_found(c, entry, changed, r, pks != nullptr, left);
  audit_run last;
  {
    std::unique_lock<std::mutex> g(c->mu);
    if (!mend) rc = repair_locked(c, g, r, pks, live, changed);
    if (rc == HS_OK) rc = audit_enqueue_locked(c, entry, pks, live, S.n_slots, last, &sl);
  }
  if (rc == HS_OK) rc = audit_collect(c, entry, changed, last);
  if (rc != HS_OK && rc != HS_ERR_ARG) return rc;
  // A repair the slot map changed under is not proved: its findings count as failed.
  const audit_run &after = rc == HS_OK ? last : r;
  rep.failed = after.failed();
  S.stats[SCRUB_FINDINGS] += scrub_items(r);
  S.stats[SCRUB_FAILED] += scrub_items(after);
  for (size_t k = 0; k < r.n_slots && !mend; k++) S.stats[SCRUB_REPAIRED] += (r.bits()[2 + k] && !after.bits()[2 + k]) ? 1 : 0;
  return HS_OK;
}
// The signature-cache slice of a tick, under S.m and whether or not the slot map is paused: the next sig_per_tick buckets of the attached
// queue's table (hs_scrub_sig_cache), wrapping at its end; a new table starts at bucket 0, and a cache that is off is skipped.  A
// correction is reported as HS_AUDIT_SIGCACHE in found, never in failed: the entry holds the re-checked byte once it is corrected.
static int scrub_sig_tick(hs_ctx *c, scrub_state &S, scrub_report &rep) {
  if (!S.sig_q) return HS_OK;
  std::lock_guard<std::mutex> ga(c->audit_mu);
  uint64_t out[HS_QUEUE_SIG_AUDIT_OUT];
  HS_TRY(sig_audit_run(
      S.sig_q, "hs_scrub",
      [&S](uint32_t buckets, uint32_t gen, sig_audit_range &r) {
        if (gen != S.sig_gen) {
          S.sig_gen = gen;
          S.sig_next = 0;
        }
        if (!buckets) return true;
        r.first = S.sig_next;
        r.n = std::min<size_t>(S.sig_per_tick, buckets - r.first);
        S.sig_next = r.first + r.n;
        if (S.sig_next >= buckets) {
          r.pass = true;
          S.sig_next = 0;
        }
        return true;
      },
      out));
  if (out[1]) rep.found |= HS_AUDIT_SIGCACHE;
  return HS_OK;
}
static void scrub_loop(hs_ctx *c) {
  scrub_state &S = c->scrub;
  pthread_setname_np(pthread_self(), "hs_scrub");  // names it in ps / top and /proc/<pid>/task/*/comm
  cudaSetDevice(c->device);
  std::unique_lock<std::mutex> l(S.m);
  while (!S.cv.wait_for(l, std::chrono::microseconds(S.period_us), [&S] { return S.stop; })) {
    scrub_report rep;
    if ((S.rc = scrub_tick(c, S, rep)) != HS_OK) return;
    if ((S.rc = scrub_sig_tick(c, S, rep)) != HS_OK) return;
    if (rep.found && S.cb) {  // without S.m: the callback may call hs_scrub_set_map
      l.unlock();
      S.cb(S.user, rep.found, rep.failed, rep.first_slot);
      l.lock();
    }
  }
}

extern "C" int hs_scrub_start(hs_ctx *c, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots, uint32_t period_us,
                              uint32_t slots_per_tick, uint32_t base_entries_per_tick, hs_scrub_cb *cb, void *user) {
  if (!c || !period_us || !slots_per_tick || !base_entries_per_tick) return fail_args(c, "hs_scrub_start", "bad argument");
  std::lock_guard<std::mutex> gl(c->scrub_life);
  scrub_state &S = c->scrub;
  if (S.th.joinable()) return fail_args(c, "hs_scrub_start", "a scrub is already running on this context (hs_scrub_stop it first)");
  {
    std::lock_guard<std::mutex> l(S.m);
    HS_TRY(scrub_map_locked(c, S, "hs_scrub_start", expect_pks, expect_live, n_slots));
    S.period_us = period_us;
    S.slots_per_tick = slots_per_tick;
    S.base_per_tick = base_entries_per_tick;
    S.cb = cb;
    S.user = user;
    S.stop = false;
    S.rc = HS_OK;
    for (auto &v : S.stats) v = 0;
  }
  try {
    S.th = std::thread(scrub_loop, c);
  } catch (const std::system_error &) {
    return fail(c, HS_ERR_NOMEM, "hs_scrub_start: no thread");
  }
  return HS_OK;
}

extern "C" int hs_scrub_set_map(hs_ctx *c, const uint8_t *expect_pks, const uint32_t *expect_live, size_t n_slots) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> l(c->scrub.m);
  return scrub_map_locked(c, c->scrub, "hs_scrub_set_map", expect_pks, expect_live, n_slots);
}

extern "C" int hs_scrub_stop(hs_ctx *c) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> gl(c->scrub_life);
  scrub_state &S = c->scrub;
  if (!S.th.joinable()) return HS_OK;
  if (S.th.get_id() == std::this_thread::get_id()) return fail_args(c, "hs_scrub_stop", "called from the scrub's callback");
  {
    std::lock_guard<std::mutex> l(S.m);
    S.stop = true;
  }
  S.cv.notify_all();
  S.th.join();
  const int rc = S.rc;
  S.rc = HS_OK;
  return rc;
}

extern "C" int hs_scrub_sig_cache(hs_ctx *c, hs_queue *q, uint32_t buckets_per_tick) {
  if (!c || (q && (q->c != c || !buckets_per_tick))) return fail_args(c, "hs_scrub_sig_cache", "bad argument");
  scrub_state &S = c->scrub;
  std::lock_guard<std::mutex> l(S.m);
  S.sig_q = q;
  S.sig_per_tick = buckets_per_tick;
  S.sig_gen = 0;
  S.sig_next = 0;
  return HS_OK;
}

extern "C" int hs_scrub_mend(hs_ctx *c, int on) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> l(c->scrub.m);  // between ticks
  c->scrub.mend = on != 0;
  return HS_OK;
}

extern "C" int hs_scrub_stats(hs_ctx *c, uint64_t out[HS_SCRUB_STATS]) {
  if (!c || !out) return HS_ERR_ARG;
  for (int k = 0; k < SCRUB_NSTATS; k++) out[k] = c->scrub.stats[k].load();
  return HS_OK;
}

// ---- explanation of a verdict (hs_explain_rec128): k_explain over the staged records, on the context's stream.  No context table is
// read and no key-cache, queue or committee state is touched, so only the staging and result buffers need the mutex.
extern "C" int hs_explain_rec128(hs_ctx *c, const hs_rec128 *recs, size_t n, uint8_t *out_why) {
  if (!c || (n && (!recs || !out_why))) return fail(c, HS_ERR_ARG, "hs_explain_rec128: bad argument");
  if (n == 0) return HS_OK;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  h2d_stage S;
  const size_t s_recs = S.add(recs, n * sizeof(hs_rec128));
  HS_TRY(ensure(c, c->out, n));
  HS_TRY(S.upload(c, c->in[0], c->stream));
  const unsigned grid = (unsigned)std::min<size_t>(blocks_for(n), (size_t)c->n_sms * 4);
  k_explain<<<grid, HS_THREADS, 0, c->stream>>>(S.ptr(s_recs), n, (uint8_t *)c->out.p.get());
  c->launches++;
  HS_CUDA(c, cudaGetLastError());
  return readback(c, {{out_why, c->out.p.get(), n}});
}

#ifdef HS_TEST_HOOKS
// Test builds only (never declared in include/hs_crypto.h, never in the product library): XORs one byte of a key slot's comb table
// (index = slot, byte_offset into its table), of the base-point table (index = entry, byte_offset into it), of a slot's key bytes
// (index = slot, byte_offset < 32) or a slot's flag byte (index = slot, byte_offset 0), on an idle context.  It cannot reach the hash
// table, the one stored value that becomes an address, so a poke can change verdicts but cannot make a kernel fault.
enum { POKE_TABLE = 0, POKE_BASE = 1, POKE_KEY = 2, POKE_FLAG = 3 };
extern "C" int hs_test_poke(hs_ctx *c, int region, size_t index, size_t byte_offset, uint8_t xor_mask) {
  if (!c) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(c->mu);
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaDeviceSynchronize());
  const size_t n = has_key_tables(c) ? c->n_keys : 0;
  uint8_t *p = nullptr;
  if (region == POKE_TABLE && index < n && byte_offset < c->a_table_entries * sizeof(ge_niels))
    p = reinterpret_cast<uint8_t *>(c->keys.atables + index * c->a_table_entries) + byte_offset;
  else if (region == POKE_BASE && index < comb_table_entries(c->cp.wb) && byte_offset < sizeof(ge_niels))
    p = reinterpret_cast<uint8_t *>(c->d_btable + index) + byte_offset;
  else if (region == POKE_KEY && index < n && byte_offset < 32)
    p = c->keys.pks + 32 * index + byte_offset;
  else if (region == POKE_FLAG && index < n && byte_offset == 0)
    p = c->keys.key_flags + index;
  if (!p) return fail_args(c, "hs_test_poke", "region, index or offset out of range");
  uint8_t v = 0;
  HS_CUDA(c, cudaMemcpy(&v, p, 1, cudaMemcpyDeviceToHost));
  v ^= xor_mask;
  HS_CUDA(c, cudaMemcpy(p, &v, 1, cudaMemcpyHostToDevice));
  return HS_OK;
}
// Arms one byte (hs_test_poke's POKE_TABLE, POKE_KEY or POKE_FLAG addressing) that c's next hs_committee_stage_register XORs in its
// staged store between the build and the proof; an index or offset past that store leaves it untouched.  One armed byte per process.
static struct {
  hs_ctx *c = nullptr;
  int region = 0;
  size_t index = 0, byte_offset = 0;
  uint8_t xor_mask = 0;
} staged_poke;
static std::mutex staged_poke_mu;
extern "C" int hs_test_poke_staged(hs_ctx *c, int region, size_t index, size_t byte_offset, uint8_t xor_mask) {
  if (!c || (region != POKE_TABLE && region != POKE_KEY && region != POKE_FLAG)) return HS_ERR_ARG;
  std::lock_guard<std::mutex> g(staged_poke_mu);
  staged_poke.c = c;
  staged_poke.region = region;
  staged_poke.index = index;
  staged_poke.byte_offset = byte_offset;
  staged_poke.xor_mask = xor_mask;
  return HS_OK;
}
// Applies and disarms the armed byte when it is c's, on the staged store K of N slots, on `stream` behind its build.
static int staged_poke_apply(hs_ctx *c, key_store &K, size_t N, size_t entries, cudaStream_t stream) {
  std::lock_guard<std::mutex> g(staged_poke_mu);
  if (staged_poke.c != c) return HS_OK;
  staged_poke.c = nullptr;
  const size_t i = staged_poke.index, off = staged_poke.byte_offset;
  uint8_t *p = nullptr;
  if (staged_poke.region == POKE_TABLE && i < N && off < entries * sizeof(ge_niels)) p = reinterpret_cast<uint8_t *>(K.atables + i * entries) + off;
  else if (staged_poke.region == POKE_KEY && i < N && off < 32) p = K.pks + 32 * i + off;
  else if (staged_poke.region == POKE_FLAG && i < N && off == 0) p = K.key_flags + i;
  if (!p) return HS_OK;
  uint8_t v = 0;
  HS_CUDA(c, cudaMemcpyAsync(&v, p, 1, cudaMemcpyDeviceToHost, stream));
  HS_CUDA(c, cudaStreamSynchronize(stream));
  v ^= staged_poke.xor_mask;
  HS_CUDA(c, cudaMemcpyAsync(p, &v, 1, cudaMemcpyHostToDevice, stream));
  return HS_OK;
}
// XORs one byte of the signature-cache entry of q that holds rec (sig | key bytes | Digest) on an idle queue: byte_offset < 128 into its
// words, 128 its flag byte.  HS_ERR_ARG when the cache is off, no entry holds rec or the offset is past the flag byte.  It changes the
// bytes a hit answers from, never seq or the round-robin counter.
extern "C" int hs_test_poke_sig(hs_queue *q, const uint8_t rec[128], size_t byte_offset, uint8_t xor_mask) {
  if (!q || !rec || byte_offset > 128) return HS_ERR_ARG;
  hs_ctx *c = q->c;
  std::lock_guard<std::mutex> g(c->mu);
  if (!q->d_sig) return fail_args(c, "hs_test_poke_sig", "the signature cache is off");
  HS_CUDA(c, cudaSetDevice(c->device));
  HS_CUDA(c, cudaDeviceSynchronize());
  std::vector<sig_bucket> t((size_t)q->sig_bmask + 1);
  HS_CUDA(c, cudaMemcpy(t.data(), q->d_sig, t.size() * sizeof(sig_bucket), cudaMemcpyDeviceToHost));
  for (size_t b = 0; b < t.size(); b++)
    for (int e = 0; e < HS_SIG_WAYS; e++) {
      const sig_entry &x = t[b].e[e];
      if (!x.seq || (x.seq & 1u) || memcmp(x.w, rec, 128)) continue;
      const size_t off = b * sizeof(sig_bucket) + e * sizeof(sig_entry) + (byte_offset < 128 ? byte_offset : offsetof(sig_entry, flags));
      uint8_t *p = reinterpret_cast<uint8_t *>(q->d_sig.get()) + off;
      const uint8_t v = reinterpret_cast<const uint8_t *>(t.data())[off] ^ xor_mask;
      HS_CUDA(c, cudaMemcpy(p, &v, 1, cudaMemcpyHostToDevice));
      return HS_OK;
    }
  return fail_args(c, "hs_test_poke_sig", "no entry holds the record");
}
#else
static int staged_poke_apply(hs_ctx *, key_store &, size_t, size_t, cudaStream_t) { return HS_OK; }
#endif
