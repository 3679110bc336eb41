/*
 * hs_crypto.h — C ABI of the H100 batch Ed25519 verification / SHA-512 digest engine.
 *
 * This is the drop-in boundary for ONE path of asonnino/hotstuff: the `crypto` crate's verify / verify_batch /
 * Digest surface.  The reference has no FFI today (it calls ed25519-dalek directly, crypto/Cargo.toml:10); each
 * entry point below names the reference interface it replaces (paths relative to the reference repo root).
 * INTEGRATION.md shows the Rust `extern "C"` binding a maintainer would add to crypto/src/lib.rs.
 *
 * Conventions
 *   - Every function returns 0 (HS_OK) when the engine ran; verdicts are in the output buffers.  Non-zero = engine
 *     failure (CUDA error, bad argument): the caller must treat every signature of that call as REJECTED
 *     (reference behaviour: any Err drops the message, consensus/src/core.rs:434-439).  There is no CPU fallback.  A
 *     host-pointer verify call that returns HS_ERR_ARG writes nothing to its output bitmaps.
 *   - Malformed inputs (S >= l, non-decompressible A or R, ...) are verdict 0, never an error.
 *   - Host-pointer entry points copy inputs to the device, run, and copy results back before returning; nothing is
 *     retained.  `_dev` entry points take device pointers and a cudaStream_t (as void*) and return after enqueueing.
 *   - A context is bound to one CUDA device.  Its host-pointer calls are thread-safe (serialised on an internal mutex).  `_dev` calls
 *     take no mutex, so they are not serialised with calls on other threads: issue them from one thread, on one stream at a time.
 *   - A host-pointer call runs after the non-deferred `_dev` verify passes enqueued earlier on the same thread on the stream last
 *     used for one (the context remembers only the latest pass, which with one stream at a time orders it after all of them): both
 *     use the context's verify scratch, so the host call's stream waits for that pass first.  The latency path (64 records or fewer
 *     whose keys all have tables, registered or learned), the self-test, the audit, repairs, staged committee changes and the scrub
 *     have scratch of their own and do not wait.
 *   - Bitmaps: bit (i & 31) of word (i >> 5) is the verdict of item i; unused high bits of the last word are 0.
 */
#ifndef HS_CRYPTO_H
#define HS_CRYPTO_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define HS_FLAG_NO_KEY_CACHE 0x10000u /* hs_ctx_create flag: never learn unregistered keys */
#define HS_OK 0
#define HS_ERR_CUDA 1
#define HS_ERR_ARG 2
#define HS_ERR_NOMEM 3
#define HS_ERR_SELFTEST 4 /* hs_self_test: a path gave a wrong answer; hs_table_audit / hs_table_repair / hs_table_mend: a table, slot or lookup entry is wrong */

/* verdict selector for the verify entry points */
#define HS_MODE_STRICT 0u /* Signature::verify semantics  = dalek verify_strict          (crypto/src/lib.rs:200-204) */
#define HS_MODE_BATCH_EQ 1u /* per-signature condition of Signature::verify_batch          (crypto/src/lib.rs:206-219) */

typedef struct hs_ctx hs_ctx;

/* One (Signature, PublicKey, Digest) triple exactly as Signature::verify receives it:
 * sig = part1 || part2 (crypto/src/lib.rs:179-182,193-198), pk = PublicKey.0 (:66), msg = Digest.0 (:22). */
typedef struct {
  uint8_t sig[64];
  uint8_t pk[32];
  uint8_t msg[32];
} hs_rec128;

/* One QC vote = (PublicKey, Signature), consensus/src/messages.rs:168 `votes: Vec<(PublicKey, Signature)>`. */
typedef struct {
  uint8_t pk[32];
  uint8_t sig[64];
} hs_vote;

/* ---- lifecycle ------------------------------------------------------------------------------------------------ */
/* device: CUDA ordinal.  Builds the base-point comb table on the GPU (default window 24 bits = 8.9 GB of HBM).
 * flags: 0 = defaults; bits 0-7 = base-point window width (even, 8..26; 26 = 10 windows in 32 GB, one addition fewer per verify), bits 8-15 = forced per-key window width
 * (8..17; 0 = widest that fits ~62 % of device memory); HS_FLAG_NO_KEY_CACHE disables the key cache (also env HS_KEY_CACHE=0). */
int hs_ctx_create(hs_ctx **out, int device, uint32_t flags);
void hs_ctx_destroy(hs_ctx *ctx);
/* Human-readable description of the last failure on this context (never NULL). */
const char *hs_last_error(const hs_ctx *ctx);
/* Key cache: when NO committee is registered, keys that show up in calls carrying key bytes are learned between calls (up to
 * 4,096 keys, 14 MB of table each, allocated on first use): the first sighting of a key takes the generic path, later
 * ones the table path.  Verdicts are identical either way.  A full cache that misses on more than half of a pass is reset
 * and relearns (validator-set rotation); there is no per-key eviction, so registering the committee remains the robust
 * choice against floods of one-off keys.  Registering switches learning off; hs_committee_register(.., 0, ..) clears the committee
 * and re-enables it.  Returns the number of keys currently cached. */
size_t hs_cached_keys(const hs_ctx *ctx);
/* Comb window widths in use: per-key tables (0 when no committee is registered) and the base-point table. */
void hs_window_bits(const hs_ctx *ctx, int *key_bits, int *base_bits);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
uint64_t hs_kernel_launches(const hs_ctx *ctx);
/* Measurement hook (bench.py's roofline): with profiling on, CUDA events bracket the k_verify_main<committee> launch of every
 * verify pass, on the stream the pass runs on; hs_profile_main_ms() waits for the last pass and returns that kernel's duration. */
int hs_profile_enable(hs_ctx *ctx, int on);
double hs_profile_main_ms(hs_ctx *ctx);
/* Pinned host memory helpers (optional; any host pointer is accepted by the host entry points). */
void *hs_host_alloc(size_t bytes);
void hs_host_free(void *p);

/* ---- Signature::verify (crypto/src/lib.rs:200-204), n independent triples -------------------------------------- */
/* Callers: Block::verify consensus/src/messages.rs:64, Vote::verify :144, Timeout::verify :258, TC::verify :312. */
int hs_verify_strict_batch(hs_ctx *ctx, const hs_rec128 *recs, size_t n, uint32_t *out_bitmap);
/* Same with an explicit verdict mode (HS_MODE_*). */
int hs_verify_rec128(hs_ctx *ctx, const hs_rec128 *recs, size_t n, uint32_t mode, uint32_t *out_bitmap);
/* Variable-length messages (PureEdDSA over the raw bytes): sig[n][64], pk[n][32], msgs concatenated, off[n+1]. */
int hs_verify_var(hs_ctx *ctx, const uint8_t *sig, const uint8_t *pk, const uint8_t *msgs, const uint64_t *off, size_t n,
                  uint32_t mode, uint32_t *out_bitmap);

/* ---- Signature::verify_batch (crypto/src/lib.rs:206-219): one digest, n votes ---------------------------------- */
/* Caller: QC::verify consensus/src/messages.rs:197.  *all_ok = 1 iff every vote parses and satisfies the
 * cofactorless equation (deterministic restatement of dalek::verify_batch, SURVEY.md App. A.3). */
int hs_verify_batch_shared_msg(hs_ctx *ctx, const uint8_t digest[32], const hs_vote *votes, size_t n, int *all_ok,
                               uint32_t *out_bitmap_or_null);

/* ---- QC::verify for many certificates in one pass (consensus/src/messages.rs:180-208) --------------------------------- */
/* preimages: n_qc x 40 bytes = hash[32] || round_le[8]; the engine computes QC::digest (messages.rs:201-208) on the GPU.
 * Vote i = (key_i, sig_i) belongs to certificate qc_idx[i]; key_i = pk[i] (32 B each) or, when pk is NULL, committee key
 * validator_idx[i].  out_qc_bitmap bit j = AND over certificate j's votes of the verify_batch condition (no votes -> 1);
 * out_vote_bitmap (nullable) = per-vote verdicts.  The stake / duplicate checks of messages.rs:182-194 stay on the host.
 * This is the view-change burst of SURVEY §3D (every Timeout carries a high_qc) as ONE engine call. */
int hs_verify_qcs(hs_ctx *ctx, const uint8_t *preimages, size_t n_qc, const uint8_t *pk_or_null, const uint32_t *validator_idx_or_null,
                  const uint8_t *sig /* n_votes x 64 */, const uint32_t *qc_idx, size_t n_votes, uint32_t *out_vote_bitmap_or_null,
                  uint32_t *out_qc_bitmap);

/* ---- TC::verify / Timeout::verify for many certificates (consensus/src/messages.rs:250-265,290-315) ------------------------ */
/* Vote i = (key_i, sig_i, high_qc_rounds[i]) of certificate tc_idx[i]; its message is SHA-512(tc_rounds[tc_idx[i]]_le ||
 * high_qc_rounds[i]_le)[..32], built and hashed ON THE GPU (messages.rs:307-311: n digests that differ in 8 bytes), judged with
 * Signature::verify (strict).  out_tc_bitmap bit j = AND over certificate j's votes (no votes -> 1).  tc_idx == NULL: vote i is
 * its own certificate (n_tc == n_votes) — the shape of n Timeout messages (Timeout::digest, messages.rs:268-275; the embedded
 * high_qc goes through hs_verify_qcs).  The stake / duplicate checks of messages.rs:292-304 stay on the host. */
int hs_verify_tcs(hs_ctx *ctx, const uint64_t *tc_rounds, size_t n_tc, const uint8_t *pk_or_null, const uint32_t *validator_idx_or_null,
                  const uint8_t *sig /* n_votes x 64 */, const uint64_t *high_qc_rounds, const uint32_t *tc_idx_or_null, size_t n_votes,
                  uint32_t *out_vote_bitmap_or_null, uint32_t *out_tc_bitmap);

/* ---- mixed groups: Block::verify for many blocks in one pass (consensus/src/messages.rs:54-76) ------------------------------ */
/* Item i signs Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i]+1])) (hashed on the GPU), belongs to group group_idx[i]
 * and is judged by mode[i] (HS_MODE_*; NULL = all strict): a block is one group holding its author signature (strict, Block::digest
 * preimage :79-90), its QC's votes (batch-eq, 40-byte preimage) and its TC's votes (strict, 16-byte preimages).
 * out_group_bitmap bit j = AND over group j's items. */
int hs_verify_groups(hs_ctx *ctx, const uint8_t *preimages, const uint64_t *pre_off /* n_msgs + 1 */, size_t n_msgs, const uint8_t *sig /* n_items x 64 */,
                     const uint8_t *pk_or_null, const uint32_t *validator_idx_or_null, const uint32_t *msg_idx, const uint32_t *group_idx,
                     const uint8_t *mode_or_null, size_t n_items, size_t n_groups, uint32_t *out_item_bitmap_or_null, uint32_t *out_group_bitmap);

/* ---- wire-format ingest: bincode ConsensusMessage frames -> the arrays hs_verify_groups consumes ------------------------------ */
/* Replaces `bincode::deserialize::<ConsensusMessage>` + the per-signature walk of Block/Vote/Timeout/TC::verify
 * (consensus/src/consensus.rs:33-39,138; crypto/src/lib.rs:94-112 PublicKey = base64 *string*; :178-182 Signature = 2 x 32 raw bytes)
 * for the crypto path: frame i (frames[off[i] .. off[i+1])) becomes group i; every signature in it becomes one item (signature,
 * decoded key bytes, preimage index, verdict mode) and every digest preimage is laid out for on-GPU hashing:
 *   Propose(Block): author item (strict, Block::digest preimage) + QC votes (batch-eq; skipped for the genesis QC) + TC votes (strict)
 *   Vote: one strict item      Timeout: author item (strict, 16-byte preimage) + high_qc votes      TC: its votes (strict)
 * Host-only, stateless, thread-safe.  Output buffers are caller-owned (hs_host_alloc() them to make the following H2D copies DMA
 * directly).  Returns HS_OK, or HS_ERR_NOMEM when a capacity is too small — n_items / n_msgs / pre_bytes then hold the required
 * sizes.  A malformed frame (truncated, bad tag, bad base64, absurd length) gets kind HS_FRAME_MALFORMED and contributes no items
 * (the reference drops it with SerializationError).  The stake / duplicate pre-checks of messages.rs stay with the caller: the
 * item ranges in hs_frame_info say which keys belong to which certificate. */
#define HS_NO_ITEM 0xffffffffu
#define HS_FRAME_MALFORMED 255
typedef struct {
  uint8_t kind;          /* ConsensusMessage tag: 0 Propose, 1 Vote, 2 Timeout, 3 TC, 4 SyncRequest; HS_FRAME_MALFORMED */
  uint8_t has_tc;        /* Block.tc is Some / the frame is a TC */
  uint8_t qc_is_genesis; /* embedded QC == QC::genesis(): not verified upstream (messages.rs:67,261) */
  uint8_t pad;
  uint32_t author_item;  /* item of the author's signature (HS_NO_ITEM for TC / SyncRequest) */
  uint32_t qc_lo, qc_hi; /* items of the embedded QC's votes [lo, hi) */
  uint32_t tc_lo, tc_hi; /* items of the TC's votes [lo, hi) */
  uint64_t round, qc_round, tc_round;
} hs_frame_info;
typedef struct {
  size_t cap_items, cap_msgs, cap_pre_bytes; /* in: capacities */
  uint8_t *sig;        /* cap_items x 64 */
  uint8_t *pk;         /* cap_items x 32 */
  uint32_t *msg_idx;   /* cap_items */
  uint32_t *group_idx; /* cap_items (= frame index) */
  uint8_t *mode;       /* cap_items: HS_MODE_* */
  uint8_t *preimages;  /* cap_pre_bytes */
  uint64_t *pre_off;   /* cap_msgs + 1 */
  size_t n_items, n_msgs, pre_bytes; /* out */
} hs_ingest_out;
int hs_ingest_consensus_frames(const uint8_t *frames, const uint64_t *off /* n + 1 */, size_t n, hs_frame_info *info /* n */, hs_ingest_out *out);

/* ---- committee mode: keys registered once per epoch (consensus/src/config.rs:28-60 Committee) ------------------- */
/* Decompresses every key and builds its comb table in HBM (window 17 bits: 94 MB, 16: 50 MB, 15: 27 MB, 14: 14 MB, 12: 4.1 MB per key).  out_valid_bitmap (nullable): bit i = key i
 * decompresses.  Replaces the per-call PublicKey::from_bytes of crypto/src/lib.rs:202,216. */
int hs_committee_register(hs_ctx *ctx, const uint8_t *pks /* N x 32 */, size_t N, uint32_t *out_valid_bitmap);
/* Incremental epoch change: validators remove_idx[] stop verifying (their indices become free), keys add_pks[] take a free
 * or spare slot (registration reserves N/16, at least 16, spare slots) and only their tables are built, in one launch; out_add_idx[i]
 * receives the index of add_pks[i] (an already-registered key returns its existing index).  Everyone else keeps index and
 * table.  HS_ERR_NOMEM when no slot is free: re-register.  Requires a registered committee.  Holds the context's mutex and drains the
 * device for the whole call, so verification waits for it; it discards a pending hs_committee_stage. */
int hs_committee_update(hs_ctx *ctx, const uint8_t *add_pks /* n_add x 32 */, size_t n_add, const uint32_t *remove_idx, size_t n_remove,
                        uint32_t *out_add_idx);
/* Staged committee change: prepare the next committee while the current one verifies, then switch it in with a short commit.
 *   - Rule: hs_committee_stage(A, R) followed by hs_committee_commit leaves the context exactly as hs_committee_update(A, none) followed
 *     by hs_committee_update(none, R): the same out_add_idx, hs_key_slots, key bytes, flag bytes, hash table, comb tables and verdicts.
 *     So added keys take free slots, lowest first, then spares; a registered key keeps its index; a key repeated in A takes one slot; a
 *     key of A whose slot is in R ends up removed; R's slots are not reused by the stage; a remove index may name any slot in use once
 *     A is in, spares included.
 *   - hs_committee_stage needs a registered committee.  Under the context's mutex it checks the arguments, picks the slots and writes
 *     the added keys' bytes; then it builds every added key's comb table in one launch and proves them all in one audit launch (the checks
 *     of hs_table_audit), on the audit's private lowest-priority stream and without the mutex, so verify queues keep launching.  It is
 *     serialised with audits and repairs, and returns once the tables are built and proved.
 *   - Until the commit, verification is exactly as before the stage: added keys are not in the committee (key-bytes calls take the
 *     generic path with the same verdicts), a committee-indexed record naming a staged index rejects, removed validators keep verifying,
 *     hs_key_slots does not change and an audit with the map from before the stage finds nothing.  A repair leaves a stage pending.
 *   - Errors: HS_ERR_NOMEM when too few free and spare slots are left (nothing is staged: use hs_committee_update); HS_ERR_ARG for a
 *     stage already pending, no registered committee, a remove index out of range, or a registration or update that ran during the
 *     stage; HS_ERR_SELFTEST when a staged table fails its proof (nothing stays staged).  Every error writes nothing.
 *   - hs_committee_commit applies the pending stage: the proved flag bytes of the added slots, the removed slots' flags cleared, then the
 *     hash table.  It builds no table.  A stage that removes slots drains the device first, as hs_committee_update does; one that only
 *     adds does not, since adding slots disturbs no launch in flight.  HS_ERR_ARG and no change when no stage is pending: none was made,
 *     or a registration or update since it discarded it.
 *   - hs_committee_discard frees the staged slots; a no-op when nothing is staged. */
int hs_committee_stage(hs_ctx *ctx, const uint8_t *add_pks /* n_add x 32 */, size_t n_add, const uint32_t *remove_idx, size_t n_remove,
                       uint32_t *out_add_idx);
int hs_committee_commit(hs_ctx *ctx);
int hs_committee_discard(hs_ctx *ctx);
/* Staged registration: build and prove a whole new key store beside the live one, then switch it in with hs_committee_commit.  Use it
 * where hs_committee_stage returns HS_ERR_NOMEM, or where the per-key window should change.
 *   - Rule: hs_committee_stage_register(P, w) followed by hs_committee_commit leaves the context exactly as hs_committee_register(P) leaves
 *     a context whose window came out as w: the same out_valid_bitmap, hs_key_slots, slot capacity (N plus N/16 spares, at least 16), key
 *     bytes, flag bytes, hash table, comb tables, hs_window_bits and verdicts on every path; the key cache is released; later
 *     hs_committee_update / hs_committee_stage calls behave as after that registration.
 *   - key_bits: 0 picks the widest window whose NEW tables alone fit in the table budget (hs_set_table_budget) and in 7/8 of the free
 *     memory with the live store still allocated, so it may be narrower than what a registration would pick after releasing the old
 *     store: discard and stage again with an explicit width to choose.  8..17: that window exactly, under the same test.  The budget
 *     bounds each store, not their sum: both stores stay resident from the stage until the commit frees the old one, so the per-key
 *     tables may use up to about twice the budget meanwhile.  A tenant sharing the device must leave room for that, or register instead.  A context created with a forced key window
 *     stages at that window.  *out_key_bits (nullable) receives the window; out_valid_bitmap (nullable): bit i = key i decompresses.
 *   - Under the context's mutex it checks the arguments and picks the geometry; then, serialised with audits, repairs, mends, scrub ticks
 *     and hs_committee_stage but without the mutex, it builds all N tables in one launch on the audit's private lowest-priority stream and
 *     proves the staged store with hs_table_audit's checks (KEY against pks, FLAG, LOOKUP, every hash entry, every comb-table entry).
 *   - Until the commit, verification is exactly as before the stage: the live tables, hs_key_slots, hs_window_bits and audits against the
 *     current map are untouched.  A context with no registered committee may stage a registration; the commit replaces its key cache.
 *   - Errors, none of which touch the live committee: HS_ERR_NOMEM when the staged store does not fit (nothing stays allocated; a budget
 *     too small for any window gives it too, where hs_committee_register would still try 8-bit windows); HS_ERR_SELFTEST when the proof
 *     fails (nothing stays staged); HS_ERR_ARG for N == 0, N >= HS_NO_KEY, key_bits outside 0 and 8..17 or unlike a forced window, a
 *     stage of either kind already pending, or a registration or update that ran during the stage.  Every error writes nothing.
 *   - hs_committee_commit applies a staged registration: it drains the device as hs_committee_register does, moves the staged store in,
 *     releases the key cache's state and starts a new slot map (the scrub pauses until hs_scrub_set_map; an audit with the old map
 *     returns HS_ERR_ARG).  It frees the old store after releasing the context's mutex.  The signature and certificate caches are kept, as
 *     for hs_committee_stage.  A registration or update since the stage discarded it: HS_ERR_ARG and no change.  hs_committee_discard
 *     frees the staged store.  A repair, mend or audit leaves a staged registration pending.
 *   - As for hs_committee_register, no `_dev` verify pass may be in flight across the commit. */
int hs_committee_stage_register(hs_ctx *ctx, const uint8_t *pks /* N x 32 */, size_t N, int key_bits, uint32_t *out_valid_bitmap,
                                int *out_key_bits);
/* Memory budget (bytes) for the per-key tables of the NEXT registration / key-cache allocation (0 = default, ~62 % of the
 * device; also env HS_TABLE_BUDGET_MB at context creation).  The engine picks the widest window that fits: e.g. 4,096 keys in
 * 18 GB -> 12-bit windows.  Lets the engine sit beside another tenant on the same GPU. */
int hs_set_table_budget(hs_ctx *ctx, size_t bytes);
/* Vote i is (validator_idx[i], sig[i]) over digests[msg_idx[i]].  msg_idx may be NULL when n_msgs == 1. */
int hs_verify_committee(hs_ctx *ctx, const uint32_t *validator_idx, const uint8_t *sig /* n x 64 */, const uint32_t *msg_idx,
                        const uint8_t *digests /* n_msgs x 32 */, size_t n_msgs, size_t n, uint32_t mode, uint32_t *out_bitmap);

/* ---- verify queue: concurrent small verifies share latency-path launches ------------------------------------------------
 * The leader's Vote::verify per incoming vote (consensus/src/core.rs handle_vote), Timeout::verify during a view change and the
 * Block author check arrive as many independent 1..64-signature requests from different tasks at once.  A queue takes them
 * without blocking and a dispatcher thread gathers EVERYTHING pending into one launch of the latency kernel whenever fewer than
 * two of its launches are in flight (continuous batching: no timers, no knobs).  Each request completes when its own records
 * are done.
 *   - hs_queue_submit copies the records into the queue's ring and returns at once: HS_ERR_NOMEM when the ring has no room for
 *     n records (retry after some requests complete), HS_ERR_ARG for n = 0, n > 64 or a bad mode.  One request = one message's
 *     signatures (a Vote, a Timeout / Block author, a small QC).
 *   - hs_queue_submit_group takes one consensus message's whole certificate as ONE request: a Block (author strict + QC votes
 *     batch-eq + TC votes strict), a Timeout with its high_qc, a TC, a QC — up to the ring's capacity, with a verdict mode per
 *     record.  It shares the ring, the dispatcher and the launches with small requests: a group whose keys are all registered
 *     costs one launch when nothing else is pending.  HS_ERR_NOMEM here means "verify it through the synchronous entry points
 *     now".
 *   - hs_queue_submit_msgs takes the same request with the signed preimages instead of their Digests (the arrays
 *     hs_ingest_consensus_frames writes for one frame), so the caller hashes nothing: the preimages go into a mapped arena beside
 *     the ring (64 bytes per ring record) and one k_queue_digests launch ahead of the verify launch, on the same stream, hashes each
 *     distinct preimage once and writes every record's Digest into the ring.  A lone device-path request costs two launches.
 *   - Verdicts equal hs_verify_rec128(ctx, recs, n, mode, ..) on the same records, bit for bit (for a group: record i equals
 *     hs_verify_rec128(ctx, &recs[i], 1, modes[i], ..)).
 *   - Device path: only when a committee is registered (hs_committee_register) and every key of the request is in it.  Any
 *     other request is run by the queue's thread through hs_verify_rec128 itself (key cache / generic kernels; a group takes
 *     at most one strict and one batch-eq call): correct, but the slow path, and it holds up the whole queue meanwhile;
 *     hs_queue_generic (off by default) verifies those requests with a queue kernel instead.  The device path has two kernels: requests of
 *     fewer than 1,002 records (every hs_queue_submit, and smaller groups) share k_verify_small launches, a block per
 *     signature, on the queue's highest-priority stream; a group of 1,002 records or more (a committee of about 1,500 or
 *     more) gets a k_verify_bulk launch of its own, a thread per signature, on a second, lower-priority stream, so a vote's
 *     launch never waits behind it.  Bulk launches do not count against the two small launches in flight.
 *   - Consumption: with a callback, it runs exactly once on the queue's thread (status HS_OK, or HS_ERR_CUDA = reject every
 *     signature of the request; bitmap = n verdict bits, valid during the call) and the ticket is released when it returns.
 *     Without one, the result is kept until ONE hs_queue_poll that reports done, or one hs_queue_wait; both return the
 *     request's status.  Reading a ticket twice, or reading a callback ticket, is HS_ERR_ARG.
 *   - hs_committee_register / hs_committee_update / hs_ctx_destroy drain the queue's launches before they touch the tables; a
 *     request submitted after one of them returns is judged against the new committee.
 *   - hs_queue_cert_cache (off by default) lets the queue verify a certificate that many requests carry once: during a view
 *     change every Timeout carries the same high_qc, and a copy that is in flight is joined and one that verified is a hit, so
 *     each Timeout puts only its author's record in the ring.  Verdicts do not change.
 *   - hs_queue_sig_cache (off by default) lets the queue's kernels verify each accepted signature once: a TC's votes are the
 *     Timeouts' author signatures the replica verified a moment earlier, so with the cache on they are probes that hit.  Verdicts
 *     do not change.
 *   - hs_queue_destroy completes every request in flight (callbacks fire) and joins the thread; hs_ctx_destroy destroys the
 *     queues still attached to the context.  hs_kernel_launches counts the queue's launches; hs_queue_stats tells them apart. */
typedef struct hs_queue hs_queue;
/* Completion callback (a function type: parameters are `hs_queue_cb *`; the parentheses keep the name from reading as a function). */
typedef void(hs_queue_cb)(void *user, size_t ticket, int status, const uint32_t *bitmap);
/* ring_records: capacity of the record ring (0 = 4,096; rounded up to a power of two, at least 64). */
int hs_queue_create(hs_ctx *ctx, size_t ring_records, hs_queue **out);
/* n = 1..64 records, mode = HS_MODE_*; callback nullable; out_ticket nullable. */
int hs_queue_submit(hs_queue *q, const hs_rec128 *recs, size_t n, uint32_t mode, hs_queue_cb *cb_or_null, void *user, size_t *out_ticket);
/* One consensus message's signatures as ONE queue request: n = 1 .. ring capacity records; record i is judged by modes[i]
 * (HS_MODE_*; NULL = all strict, as in hs_verify_groups).  HS_ERR_ARG: n = 0, n > ring capacity, a mode byte > 1.
 * HS_ERR_NOMEM: no room right now (back-pressure).  Completion, tickets, poll / wait / callback exactly as hs_queue_submit; the
 * bitmap holds n bits (poll / wait: (n + 31) / 32 words). */
int hs_queue_submit_group(hs_queue *q, const hs_rec128 *recs, size_t n, const uint8_t *modes_or_null, hs_queue_cb *cb_or_null, void *user,
                          size_t *out_ticket);
/* One consensus message's signatures as ONE queue request, with the signed preimages instead of their Digests: record i is
 * (sig[i], pk[i]) over Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1])) = SHA-512(..)[..32], hashed ON THE GPU,
 * judged by modes[i] (HS_MODE_*; NULL = all strict).  Exactly the arrays hs_ingest_consensus_frames writes for one frame.
 * n = 1 .. ring capacity, n_msgs >= 1 (a preimage no record names is not hashed).  HS_ERR_ARG: bad sizes / offsets, msg_idx[i] >= n_msgs, a mode byte > 1, or more
 * preimage bytes than the queue's preimage arena holds (64 bytes per ring record, offsets and indices included).  HS_ERR_NOMEM: no
 * ring or arena room right now (back-pressure).  Completion, tickets, poll / wait / callback exactly as hs_queue_submit_group. */
int hs_queue_submit_msgs(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off /* n_msgs + 1 */, size_t n_msgs,
                         const uint8_t *sig /* n x 64 */, const uint8_t *pk /* n x 32 */, const uint32_t *msg_idx /* n */,
                         const uint8_t *modes_or_null, size_t n, hs_queue_cb *cb_or_null, void *user, size_t *out_ticket);
/* Non-blocking: *done = 0 (come back later) or 1 (out_bitmap holds the verdicts, ticket consumed, returns the request's status). */
int hs_queue_poll(hs_queue *q, size_t ticket, int *done, uint32_t *out_bitmap);
/* Blocks until the request is done; consumes the ticket and returns the request's status. */
int hs_queue_wait(hs_queue *q, size_t ticket, uint32_t *out_bitmap);
/* Counters since hs_queue_create (each a uint64_t): [0] k_verify_small launches, [1] records they carried (riders included),
 * [2] k_verify_bulk launches, [3] records they carried, [4] slow-path requests, [5] their records. */
#define HS_QUEUE_STATS 6
int hs_queue_stats(hs_queue *q, uint64_t out[HS_QUEUE_STATS]);
/* [0] k_queue_digests launches, [1] preimages hashed, [2] preimage bytes hashed, [3] hs_queue_submit_msgs requests. */
#define HS_QUEUE_DIGEST_STATS 4
int hs_queue_digest_stats(hs_queue *q, uint64_t out[HS_QUEUE_DIGEST_STATS]);
/* Certificate cache of hs_queue_submit_group / hs_queue_submit_msgs.  A span is the HS_MODE_BATCH_EQ records of one request that
 * sign the same message (the 32-byte Digest for submit_group, the preimage bytes for submit_msgs; the two never match), at least
 * two of them: a QC's votes.  Strict records are never cached.  A span matches only a span with the same kind, message and
 * (pk, sig) of every record in the same order, byte for byte.  A span whose records all verified is kept: a later identical span
 * is a hit and answers 1 for each of its records.  An identical span still pending or in flight in an earlier request is joined:
 * the later request takes that request's bits for it and its status (HS_ERR_CUDA propagates).  Hit and joined records take no
 * ring slot and their preimages no arena bytes, so HS_ERR_NOMEM and the ring-capacity and arena-size HS_ERR_ARG apply to the
 * records that enter the ring (a Timeout whose high_qc hits costs one record).  A request answered entirely from the cache still
 * gets a ticket and completes on the queue's thread.  Verdicts are bit for bit those of the same request with the cache off.
 * 0 = off (the default: every request behaves exactly as without this call). Otherwise keep up to max_bytes of verified certificates
 * (the key bytes: 9 + message length + 96 per record), least recently used first out. */
int hs_queue_cert_cache(hs_queue *q, size_t max_bytes);
#define HS_QUEUE_CERT_STATS 6
/* [0] spans looked up, [1] cache hits, [2] in-flight joins, [3] records answered without verifying them,
 * [4] spans inserted, [5] bytes held now */
int hs_queue_cert_stats(hs_queue *q, uint64_t out[HS_QUEUE_CERT_STATS]);
/* Signature cache of the queue's device path: a table in HBM of the records its kernels accepted, so a signature the node already
 * verified (a Timeout's author vote, then the same vote inside the TC and the Block carrying it) costs a probe, not a verify.
 *   - A cached record is (sig[64], pk[32], msg[32]) with the KEY BYTES, never a committee index (hs_committee_update reuses
 *     indices), mapped to the record's flag byte (both verdicts), so a hit answers either mode exactly: a small-order key accepted
 *     under batch-eq is still rejected strict.  A hit needs all 128 bytes equal; verdicts are bit for bit those of the same request
 *     with the cache off, and committee changes do not flush the cache (a record's flags depend only on its bytes).
 *   - Only records that verified under batch-eq with a registered key are inserted; rejected records are verified every time.
 *   - Only device-path records take part: slow-path requests and riders neither probe nor insert.  Hit records keep their ring
 *     slot and their place in the launch (only the curve arithmetic is skipped); the ring, arena, completion, tickets and
 *     hs_queue_stats do not change.
 * entries: 0 = off (the default: the queue launches exactly the kernels it launches without this call); otherwise the table holds
 * at least `entries` records (buckets of 4 entries of 144 bytes, a power of two of buckets), at most 2^26.  Changing the size or
 * turning it off first drains the queue's launches in flight and starts from an empty table.  HS_ERR_NOMEM: no device memory. */
int hs_queue_sig_cache(hs_queue *q, size_t entries);
#define HS_QUEUE_SIG_STATS 5
/* Counters of completed launches: [0] records probed, [1] hits, [2] inserts, [3] inserts that evicted a live entry,
 * [4] entries held now */
int hs_queue_sig_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_STATS]);
/* Sharing of q's signature cache with the synchronous verify calls on q's context and with q's batch lane.  A TC's votes are the
 * Timeouts' author signatures; when the Timeouts came through the queue, a TC or Block above GROUP_MAX_SIGS verified synchronously,
 * or a collected burst on the batch lane, then answers those records from the same table instead of verifying them again.
 *   - on = 0 is the default: every call launches exactly the kernels it launches without this call.
 *   - Taking part once on = 1, they probe q's table and fill it: the host-pointer calls hs_verify_strict_batch, hs_verify_rec128,
 *     hs_verify_batch_shared_msg, hs_verify_qcs, hs_verify_tcs and hs_verify_groups on q's context, when their pass runs the committee
 *     kernel (k_verify_main<committee>); and q's batch-lane passes.
 *   - Not taking part: the latency path of 64 records or fewer; every `_dev` entry point (deferred mode, the peer all-gather);
 *     hs_verify_msgs, hs_verify_var and hs_verify_committee; hs_self_test, the table audit and the repair; and the calls q's own
 *     dispatcher makes for slow-path requests (slow-path requests and riders neither probe nor insert, as above).
 *   - Probe: the table's rule, all 128 bytes equal (sig, the registered key's bytes, the Digest); a committee-indexed record uses its
 *     slot's key bytes.  Records whose key is not registered take the generic side pass and neither probe nor insert; a record whose
 *     committee slot is out of service (removed by hs_committee_update, or being rebuilt by hs_table_repair) is verified, and so
 *     rejected, exactly as with sharing off.
 *   - Insert: only a record judged in STRICT mode whose flags have HS_F_EQ, with its whole flag byte, so a hit answers both modes.
 *     Strict records are the ones a node meets again (a Timeout author's signature returns in the TC and in the Block carrying it);
 *     a Block's QC votes (batch-eq) do not, and inserting them would evict those every round.
 *   - Verdicts are bit for bit those of the same call with sharing off.
 *   - HS_ERR_ARG when q's signature cache is off or another queue of the context already shares.  hs_queue_sig_cache(q, 0) and
 *     hs_queue_destroy(q) end the sharing; a resize keeps it, with the new table, after the lane passes in flight and under the
 *     context's lock, which the synchronous calls hold until their results are back.  A table repair empties the shared table.
 *   - hs_queue_sig_stats keeps counting the queue's ring kernels only, except [4] (entries held), which includes shared inserts.
 *   - hs_multi_* calls run member entry points: a member whose queue shares takes part. */
int hs_queue_sig_share(hs_queue *q, int on);
#define HS_QUEUE_SIG_SHARE_STATS 5
/* Counters of the shared passes whose results are back: [0] records probed, [1] hits, [2] inserts, [3] inserts that evicted a live
 * entry, [4] shared passes */
int hs_queue_sig_share_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_SHARE_STATS]);
/* Audit of q's signature cache: every held entry of buckets [first_bucket, first_bucket + n_buckets) re-checked from its 128 stored
 * bytes, and the flag bytes that disagree corrected.  A hit answers from the stored flag byte with no check at all, so a flipped bit
 * there is a false accept (a batch-eq-only record answered strict) or a false reject that lasts until the entry is evicted.
 *   - Check: a thread per entry reads it as one version by the probes' rule (an entry being written, or changed between the reads, is
 *     skipped), computes k = SHA-512(R || A || Digest) and hs_explain_rec128's mask with no table of any kind (no comb table, key slot
 *     or base-point table), and derives from the mask the flag byte every verify path writes for that record.
 *   - Correction: an entry whose flag byte differs gets the derived byte under the writers' protocol; one a writer claimed meanwhile
 *     holds a newer record and is skipped.  A corrected entry's hits then answer exactly what a verify answers, reject included.
 *     Entries are never emptied or evicted by the audit, and the probe and insert paths are unchanged.
 *   - n_buckets = 0: from first_bucket to the end of the table (the whole table with first_bucket 0).  HS_ERR_ARG writes nothing: q or
 *     out NULL, the cache off, or a range that leaves the table.
 *   - out: [0] entries held (re-checked), [1] corrected, [2] skipped, [3] the first corrected position (bucket * 4 + way; UINT64_MAX:
 *     none), [4] its stored flag byte, [5] its derived flag byte, [6] its HS_WHY_* mask ([4..6] are 0 with no correction).
 *   - Synchronous.  The kernel runs on the table audit's private stream of the lowest priority, on at most a quarter of the SMs, and
 *     takes hs_table_audit's turn (audits, repairs, stages, commits and scrub ticks of the context run one at a time); the context's
 *     mutex is held only to read the table and enqueue, so the queue keeps launching beside it.  hs_queue_sig_cache (a resize, off,
 *     or the flush of hs_table_repair) waits for an audit in flight before its table goes.
 *   - hs_scrub_sig_cache runs it a slice per scrub tick. */
#define HS_QUEUE_SIG_AUDIT_OUT 7
int hs_queue_sig_audit(hs_queue *q, size_t first_bucket, size_t n_buckets, uint64_t out[HS_QUEUE_SIG_AUDIT_OUT]);
#define HS_QUEUE_SIG_AUDIT_STATS 5
/* Counters over hs_queue_sig_audit calls and scrub slices: [0] audits, [1] entries re-checked (held), [2] corrected, [3] skipped,
 * [4] full passes of the table */
int hs_queue_sig_audit_stats(hs_queue *q, uint64_t out[HS_QUEUE_SIG_AUDIT_STATS]);
/* Generic-key device path of the queue.  0 = off (the default: the queue launches exactly the kernels it launches without this
 * call, and a request the committee path cannot serve runs synchronously on the queue's thread).  On: such a request (no committee
 * registered, or any key of the request outside it) is verified on the GPU instead, by k_queue_generic on the queue's
 * lower-priority stream (a thread per record: decompress A, a radix-16 window for [k](-A), the base comb for [S]B), so it no longer
 * holds up the dispatcher or the other requests' launches.  At most one such launch is in flight; it takes every generic request
 * pending, and it does not count against the two small launches in flight.  preimage requests get their Digests from a
 * k_queue_digests launch ahead of it on the same stream.
 *   - Verdicts are bit for bit those of the same request with the option off, i.e. hs_verify_rec128 per record in its mode.
 *   - Requests the generic path takes do not count in hs_queue_stats [4..5] (they count in hs_queue_generic_stats).
 *   - Turning the option off drains the generic launches in flight; requests still waiting for one then take the slow path.
 *   - Their records neither probe nor fill the signature cache: only device-path records with a registered key take part.  The
 *     certificate cache works on them as on any request.  The key cache does not learn from queue requests.
 * HS_ERR_NOMEM: no pinned host memory for the slot list (first use). */
int hs_queue_generic(hs_queue *q, int on);
#define HS_QUEUE_GENERIC_STATS 3
/* [0] k_queue_generic launches, [1] records they carried, [2] requests */
int hs_queue_generic_stats(hs_queue *q, uint64_t out[HS_QUEUE_GENERIC_STATS]);
/* Batch lane: a whole hs_verify_groups pass as ONE non-blocking queue request (a 10,000-validator Block, a view-change burst of
 * Timeouts, many ingested frames), verified by the throughput kernels of hs_verify_groups on the lane's own stream and scratch.  The
 * context's mutex is held only while the pass's launches are enqueued, so the queue's vote launches and the synchronous entry
 * points go on meanwhile.  Batch requests never enter the ring, take no part in the certificate or signature caches and do not
 * count in the other queue counters; they run one pass at a time, in submit order.
 * max_items / max_bytes bound one request (items; bytes of its arena region: offsets, preimages, signatures, keys, indices, modes,
 * result words).  0, 0 = off (the default).  Resizing or turning it off first waits for every batch request already submitted.
 * HS_ERR_NOMEM: no pinned host or device memory (the lane is then off). */
int hs_queue_batch(hs_queue *q, size_t max_items, size_t max_bytes);
/* hs_verify_groups as ONE non-blocking queue request.  The arrays and meaning are those of hs_verify_groups with key bytes.
 * Item i is (sig[i], pk[i]) over Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1])), in group group_idx[i],
 * judged by modes[i] (NULL = all strict).  Group and item bits equal hs_verify_groups on the same arrays, bit for bit, with or
 * without a registered committee (without one every item takes the generic kernel; the lane never teaches the key cache).
 * Completion, tickets, poll / wait / callback work as for hs_queue_submit_group.  The bitmap has ceil(n_groups / 32) words of
 * group bits, then ceil(n_items / 32) words of item bits.  A group with no items is 1.
 * HS_ERR_ARG: the lane is off; n_items or n_groups is 0; bad offsets; msg_idx >= n_msgs; group_idx >= n_groups; a mode byte > 1;
 * more items or region bytes than the lane's limits.  HS_ERR_NOMEM: no arena room right now (back-pressure). */
int hs_queue_submit_batch(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off, size_t n_msgs, const uint8_t *sig,
                          const uint8_t *pk, const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *modes_or_null,
                          size_t n_items, size_t n_groups, hs_queue_cb *cb_or_null, void *user, size_t *out_ticket);
#define HS_QUEUE_BATCH_STATS 5
/* Counters of completed batch passes: [0] batch passes, [1] items, [2] groups, [3] preimage bytes hashed, [4] items whose key was
 * outside the committee (every item when no committee is registered) */
int hs_queue_batch_stats(hs_queue *q, uint64_t out[HS_QUEUE_BATCH_STATS]);
/* Explain lane: hs_explain_rec128 as a non-blocking queue request, for the records of a message a node has already seen rejected.  The
 * synchronous call holds the context's mutex for its whole re-check (about 1.4 ms), and every queue launch needs that mutex to enqueue;
 * the lane holds it only while its launch is enqueued, so explaining junk from a peer no longer holds up the votes.
 *   - One k_queue_explain launch takes every explain request pending when it is launched (a thread per record, the re-check of
 *     hs_explain_rec128), on the lane's own stream at the device's lowest priority; at most one is in flight, and it does not count
 *     against the two small launches in flight.  Its grid is at most one block of 128 threads per 4 SMs (33 blocks, 4,224 records per
 *     wave on a 132-SM H100), grid-stride beyond that, so a large request leaves three quarters of the SMs to the verify launches.
 *   - The lane reads no context table (no comb table, key slot, key flag or hash table, and not the base-point table) and takes no ring
 *     slot: explain records live in the lane's own mapped arena.  Committee changes, audits and repairs therefore neither drain it nor
 *     change its answers.
 *   - Isolation: explain requests take no part in the certificate or signature caches, do not teach the key cache and do not move
 *     hs_queue_stats, hs_queue_digest_stats, hs_queue_generic_stats or hs_queue_batch_stats.  hs_queue_destroy completes every explain
 *     request in flight (callbacks fire).
 * max_records / max_bytes bound one request (records; bytes of its arena region: 128 per record, plus for the preimage form the offsets,
 * indices and preimage bytes, plus the why bytes, each section rounded up to 16, plus 16).  0, 0 = off (the default: the queue launches
 * exactly the kernels it launches without this call).  Resizing or turning it off first waits for every explain request already
 * submitted.  HS_ERR_NOMEM: no pinned host or device memory (the lane is then off). */
int hs_queue_explain(hs_queue *q, size_t max_records, size_t max_bytes);
/* hs_explain_rec128(ctx, recs, n, ..) as ONE non-blocking queue request: the mask of record i is byte for byte what that call returns.
 * Completion, tickets, poll / wait / callback work as for hs_queue_submit_group, but the uint32_t words hold the why bytes packed
 * little-endian: byte i (bits 8 (i & 3) .. 8 (i & 3) + 7 of word i >> 2) is record i's HS_WHY_* mask, and there are (n + 3) / 4 words
 * (unused bytes of the last word are 0).  A failed request (status HS_ERR_CUDA) has all-zero words: it explains nothing.
 * HS_ERR_ARG: the lane is off, n = 0, NULL recs, or more records or region bytes than the lane's limits.  HS_ERR_NOMEM: no arena room
 * right now (back-pressure: explain later, or not at all).  An explanation is advisory: a refused request never changes a verdict. */
int hs_queue_submit_explain(hs_queue *q, const hs_rec128 *recs, size_t n, hs_queue_cb *cb_or_null, void *user, size_t *out_ticket);
/* The same with the signed preimages instead of their Digests, in the arrays of hs_queue_submit_msgs without the modes: record i is
 * (sig[i], pk[i]) over Digest = SHA-512(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]))[..32], hashed on the GPU by the
 * record's own thread.  Its mask equals hs_explain_rec128 on the record built with that Digest.  HS_ERR_ARG as hs_queue_submit_explain,
 * and for the checks of hs_queue_submit_msgs: bad offsets, n_msgs = 0, msg_idx[i] >= n_msgs. */
int hs_queue_submit_explain_msgs(hs_queue *q, const uint8_t *preimages, const uint64_t *pre_off /* n_msgs + 1 */, size_t n_msgs,
                                 const uint8_t *sig /* n x 64 */, const uint8_t *pk /* n x 32 */, const uint32_t *msg_idx /* n */, size_t n,
                                 hs_queue_cb *cb_or_null, void *user, size_t *out_ticket);
#define HS_QUEUE_EXPLAIN_STATS 3
/* Counters of completed explain launches: [0] k_queue_explain launches, [1] records, [2] requests */
int hs_queue_explain_stats(hs_queue *q, uint64_t out[HS_QUEUE_EXPLAIN_STATS]);
void hs_queue_destroy(hs_queue *q);

/* ---- Digest surface: out[i] = SHA-512(data[off[i] .. off[i+1]))[0..32] ------------------------------------------ */
/* Replaces Sha512::digest(..)[..32] at mempool/src/processor.rs:30 and consensus/src/messages.rs:81,151,203,270,308. */
int hs_digest32_batch(hs_ctx *ctx, const uint8_t *data, const uint64_t *off, size_t n, uint8_t *out /* n x 32 */);

/* ---- reference-shaped end-to-end call: verdict_i = Signature::verify(Digest(msg_i), key_i) ----------------------- */
/* n fixed-size messages (msg_len bytes each, concatenated); key_i = pk[i] (pk != NULL) or committee key validator_idx[i].
 * Computes the 32-byte Digest on the GPU (mempool/src/processor.rs:30 / consensus/src/messages.rs digests) and verifies
 * over it, overlapping the host->device copy of one chunk with the kernels of the previous one. */
int hs_verify_msgs(hs_ctx *ctx, const uint8_t *sig /* n x 64 */, const uint8_t *pk_or_null /* n x 32 */, const uint32_t *validator_idx_or_null,
                   const uint8_t *msgs, size_t msg_len, size_t n, uint32_t mode, uint32_t *out_bitmap);

/* ---- known-answer self-test: every device path at this context's table geometry ------------------------------------------
 * A node has no CPU verifier behind the engine, and its table geometry is chosen at run time (base window from hs_ctx_create, per-key
 * window from the table budget and free memory).  This call drives every kernel below on private scratch and compares the answers with
 * ones compiled into the library (the golden vectors: RFC 8032, the reference crate's test signatures, adversarial and small-order
 * cases, the SHA-512 known answers).  Call it at start-up, after hs_committee_register: a failure means this box gives wrong verdicts,
 * not an error code, and the engine must not be used.
 *   - recs == NULL: the built-in set (expect == NULL, n == 0).  Otherwise the caller's n (1 .. 4,096) records with their expected
 *     verdicts run through every verify path: expect[i] bit 0 = the strict verdict, bit 1 = the batch-eq verdict.  The Digest,
 *     k_queue_digests and signer paths run only with the built-in set.  Built-in vectors whose message is not 32 bytes take only the
 *     variable-length path.
 *   - key_bits: 0 = the per-key window in use (the registered committee's, or the key cache's when it holds tables; with neither,
 *     the window registering the set's keys would pick under the current budget), or 8 .. 17 to force one.  The base-point table is
 *     always the context's own.  The committee paths use scratch tables for the set's distinct keys, built at that window (the 39
 *     distinct keys of the built-in set: about 0.3 GB at 13 bits, 3.7 GB at 17) and released before the call returns.
 *   - Returns HS_OK with *out_failed_paths = 0; HS_ERR_SELFTEST with one HS_SELFTEST_* bit per failing path, hs_last_error naming the
 *     first mismatch (path, vector name or record index, got and expected bits); HS_ERR_ARG for bad sizes, recs without expect, an
 *     expect byte above 3 or key_bits out of range; HS_ERR_NOMEM when the scratch tables do not fit in device memory.
 *   - Isolation: holds the context's mutex and runs on private streams; the registered committee, the key cache and its learning, the
 *     deferred scratch sets, the peer route, profiling and every verify queue (ring, caches, counters, stats) are not touched, so
 *     queues may keep working meanwhile.  Its launches count in hs_kernel_launches.  Like every host-pointer entry point it must not
 *     be mixed with deferred `_dev` passes in flight. */
#define HS_SELFTEST_DIGEST (1u << 0)          /* k_digest32 */
#define HS_SELFTEST_DIGEST_FIXED (1u << 1)    /* k_digest32_fixed */
#define HS_SELFTEST_DIGEST_LONG (1u << 2)     /* k_digest32_long */
#define HS_SELFTEST_GENERIC (1u << 3)         /* k_verify_main<generic> on packed records + k_verify_finish, both modes */
#define HS_SELFTEST_VAR (1u << 4)             /* the same over variable-length messages */
#define HS_SELFTEST_COMMITTEE (1u << 5)       /* k_verify_main<committee> with committee indices + k_verify_finish, both modes */
#define HS_SELFTEST_LOOKUP (1u << 6)          /* k_key_lookup + k_verify_main<committee>, a key outside the table on the side-stream pass */
#define HS_SELFTEST_MODES (1u << 7)           /* k_verify_finish_modes, mixed mode bytes */
#define HS_SELFTEST_SMALL (1u << 8)           /* k_verify_small */
#define HS_SELFTEST_SMALL_CACHE (1u << 9)     /* k_verify_small with a signature table, empty then filled */
#define HS_SELFTEST_BULK (1u << 10)           /* k_verify_bulk */
#define HS_SELFTEST_BULK_CACHE (1u << 11)     /* k_verify_bulk with a signature table, empty then filled */
#define HS_SELFTEST_QUEUE_GENERIC (1u << 12)  /* k_queue_generic */
#define HS_SELFTEST_QUEUE_DIGESTS (1u << 13)  /* k_queue_digests */
#define HS_SELFTEST_SIGN (1u << 14)           /* k_keygen + k_sign_digests */
#define HS_SELFTEST_VERIFY_PATHS 0x1ff8u      /* GENERIC .. QUEUE_GENERIC: the paths caller records run through */
int hs_self_test(hs_ctx *ctx, int key_bits, const hs_rec128 *recs_or_null, const uint8_t *expect_or_null, size_t n, uint32_t *out_failed_paths);

/* ---- audit of the live key tables: every comb-table entry, key slot and lookup entry against the key it must hold ------------------
 * hs_self_test proves the kernels on scratch tables; this call checks the state the node actually verifies against, which lives for the
 * whole process: the per-key comb tables, the slot -> key bytes array with its flags, the device hash table from key bytes to slot, and
 * the base-point table.  A slot reached from key X's bytes whose table holds multiples of key Y would accept Y's signatures as X's, so
 * call it at start-up (after hs_self_test), after every committee change, and periodically on a live node.
 *   - Tables: entry 0 of every window is exactly (1, 1, 0); every coordinate is canonical; 2 xy2d == d ((y+x)^2 - (y-x)^2); entry m is
 *     entry m - 1 plus entry 1 of its window; entry 1 of window i + 1 is twice entry 2^(w-1) of window i; entry 1 of window 0 is -A,
 *     decompressed from the slot's stored bytes (B for the base-point table).  By induction every entry is the multiple it must be.
 *   - Slots: KEY compares the stored bytes and the engine's liveness with the caller's map; FLAG checks the device flag byte against the
 *     liveness and the key's decompression; LOOKUP probes the device hash table with every live slot's bytes (it must reach a live slot
 *     with those bytes: registration keeps the first of duplicated keys) and checks that every hash entry names a live slot its own bytes
 *     reach.  A live slot whose key does not decompress has no table to check.
 *   - n_slots must equal hs_key_slots(ctx).  expect_pks (n_slots x 32, nullable) is the caller's index -> key map, for example the
 *     registration order updated with every out_add_idx; NULL checks the engine against itself.  expect_live (one bit per slot, nullable:
 *     every slot live) is compared with the engine's liveness whenever either expectation is given.  Key-cache tables take expect_pks == NULL.
 *     The base-point table is always checked; a context without per-key tables checks only it, with n_slots = 0.
 *   - Returns HS_OK with *out_failed = 0; HS_ERR_SELFTEST with the HS_AUDIT_* bits OR-ed into *out_failed, each slot's bits in
 *     out_slot_bits (nullable) and hs_last_error naming the first finding (slot, class, window and entry for a table finding).
 *     HS_ERR_ARG writes nothing: bad pointers, n_slots != hs_key_slots, expect_pks for key-cache tables, or key tables that changed while
 *     the audit ran (a registration, update or key-cache build: call it again).  HS_ERR_NOMEM / HS_ERR_CUDA as elsewhere.
 *   - Isolation: the context's mutex is held only to check the arguments, snapshot the slots and enqueue; the kernels run on a private
 *     stream of the lowest priority and the call waits for them without the mutex, so verify queues keep launching.  Reads every table and
 *     mirror and writes none; the verify queues, their caches and counters, the deferred scratch and the peer route are not touched.  Its
 *     launches count in hs_kernel_launches.  Audits of one context run one at a time.  `_dev` verify passes take no mutex and may grow
 *     the key cache, so they must not overlap an audit of the same context. */
/* Key slots in use: the registered committee's (N plus the spare slots hs_committee_update has taken, freed ones included), or the
 * key cache's learned keys; 0 when the context holds no per-key tables. */
size_t hs_key_slots(const hs_ctx *ctx);
#define HS_AUDIT_KEY    (1u << 0) /* the slot's stored key bytes, or whether it is live, differ from the caller's expectation */
#define HS_AUDIT_FLAG   (1u << 1) /* the slot's device flag byte disagrees with its liveness and with whether its key decompresses */
#define HS_AUDIT_LOOKUP (1u << 2) /* the device hash table does not take the slot's key bytes to it (or to a live slot with the same
                                     bytes), or a hash entry names this slot although it is not live */
#define HS_AUDIT_TABLE  (1u << 3) /* an entry of the slot's comb table is not the multiple of -A it must hold */
#define HS_AUDIT_BASE   (1u << 4) /* out_failed only: an entry of the base-point table is not the multiple of B it must hold */
#define HS_AUDIT_SIGCACHE (1u << 5) /* a scrub callback's found only: the tick corrected a signature-cache entry (hs_scrub_sig_cache) */
int hs_table_audit(hs_ctx *ctx, const uint8_t *expect_pks_or_null /* n_slots x 32 */, const uint32_t *expect_live_or_null /* bitmap */,
                   size_t n_slots, uint8_t *out_slot_bits_or_null /* n_slots */, uint32_t *out_failed);

/* ---- repair of what the audit finds: the failing key slots, lookup entries and the base-point table, rebuilt in place -------------
 * Runs hs_table_audit, repairs every finding, and proves the result with a complete audit.  The arguments are hs_table_audit's, with
 * its rules (n_slots == hs_key_slots, expect_pks == NULL for key-cache tables).  What a slot must hold comes from one authority: the
 * caller's map when expect_pks / expect_live are given, otherwise the engine's host mirror; never from the device bytes.
 *   - A slot with a KEY, FLAG or TABLE finding that the authority holds live gets the authority's key bytes, a rebuilt comb table and a
 *     rebuilt flag byte; one it holds dead is taken out of service, as hs_committee_update's removal would.  The device hash table is
 *     rebuilt from the authority (all a LOOKUP finding needs); a BASE finding rebuilds the base-point table.
 *   - While a committee's slots are rebuilt, verification goes on: the slots are first taken out of service (their key bytes miss the
 *     committee and take the generic path with correct verdicts; committee-indexed calls naming them reject), rebuilt and proven by the
 *     audit's checks on the audit's private lowest-priority stream without the context's mutex, and put back one by one as each passes.
 *     A slot that fails stays out of service and is reported.  Key-cache slots, and the base-point table, are rebuilt with the mutex
 *     held and the device drained: verification waits for them.
 *   - Any finding empties the signature cache and the certificate cache of every verify queue of the context (their completed entries;
 *     requests in flight complete as they would), so nothing accepted against a wrong table is answered from a cache.
 *   - *out_found: the classes the first audit found, out_slot_bits (nullable): its per-slot bits (the slots repaired), *out_failed: the
 *     classes the final audit still finds.  HS_OK iff *out_failed == 0; otherwise HS_ERR_SELFTEST and hs_last_error names the first
 *     residual finding, worded as hs_table_audit words it.  On a clean context it is one audit and changes nothing.
 *   - HS_ERR_ARG writes nothing: bad pointers, the audit's argument errors, or key tables that changed during the repair (a
 *     registration or update from another thread: the slots it left to the repair are back in service; call it again).
 *   - Repairs and audits of one context run one at a time; `_dev` verify passes must not overlap a repair, as for an audit.  A
 *     multi-device context is repaired member by member (hs_multi_member) with the same map. */
int hs_table_repair(hs_ctx *ctx, const uint8_t *expect_pks_or_null /* n_slots x 32 */, const uint32_t *expect_live_or_null /* bitmap */,
                    size_t n_slots, uint8_t *out_slot_bits_or_null /* n_slots */, uint32_t *out_found, uint32_t *out_failed);

/* ---- mend of corrupt comb-table entries in place: no drain, no slot out of service -------------------------------------------
 * Runs hs_table_audit, also noting the windows that hold its TABLE and BASE findings, recomputes those windows into a bounded scratch
 * buffer with the build's arithmetic, and stores only the entries whose bytes differ from the fresh build's.  A correct entry is never
 * written; a wrong one is overwritten once with the right bytes.  A verify that gathers an entry while it is stored reads the old value,
 * the new one or a mix of the two, and each is wrong only where the table already was, so verification goes on throughout and the
 * slot stays in service.  Then the mended windows are audited again (the base-point table's windows with the window after each, the
 * mended slots' whole tables), and, if any entry was rewritten, every verify queue's signature and certificate caches are emptied as
 * hs_table_repair empties them.  The arguments are hs_table_audit's, with its rules.
 *   - What is mended: BASE findings (the anchor B is a constant), and the TABLE findings of a slot whose only class is TABLE.  A slot whose
 *     anchor (entry 1 of window 0) fails is mended only with expect_pks given: without a map, key bytes that changed but still
 *     decompress look exactly like a bad anchor, and a table rebuilt from them would hold another key's multiples.  KEY, FLAG and LOOKUP
 *     findings, and the slots that carry them, are left untouched.
 *   - *out_found: the classes the locating audit found; out_slot_bits (nullable): its per-slot bits; *out_left: the classes left, i.e.
 *     not mendable or still failing the second audit.  HS_OK iff *out_left == 0; otherwise HS_ERR_SELFTEST, and hs_table_repair then
 *     finds only what is left.  On a clean context it is one audit and writes nothing.
 *   - Isolation: it takes the audit's turn (serialised with hs_table_audit, hs_table_repair, the committee stage and commit and the scrub's
 *     ticks) and holds the context's mutex only to snapshot, to enqueue and to empty the caches; its kernels run on the audit's
 *     lowest-priority stream.  It never drains the device and never changes a slot's service state.  Its staging (65 entries of 96
 *     bytes per thread of one launch, 211 MB on a 132-SM device) is allocated on first use and kept with the context.
 *   - HS_ERR_ARG writes nothing: the audit's argument errors, or key tables that changed between the audit and the stores (a
 *     registration, update, commit or key-cache change: nothing was stored; call it again).  A change after the stores were enqueued
 *     waits for them before it writes.  `_dev` verify passes must not overlap a mend, as for an audit.
 *   - A multi-device context is mended member by member (hs_multi_member) with the same map, as it is repaired. */
int hs_table_mend(hs_ctx *ctx, const uint8_t *expect_pks_or_null /* n_slots x 32 */, const uint32_t *expect_live_or_null /* bitmap */,
                  size_t n_slots, uint8_t *out_slot_bits_or_null /* n_slots */, uint32_t *out_found, uint32_t *out_left);
/* calls (the scrub's mends included), windows recomputed, entries rewritten, windows left (flagged but not mended, or failing the
 * second audit), slots left to hs_table_repair, cache flushes */
#define HS_MEND_STATS 6
int hs_table_mend_stats(hs_ctx *ctx, uint64_t out[HS_MEND_STATS]);

/* ---- scrub of the live key tables: the audit and repair above, a bounded slice at a time, on an engine-owned thread -------------
 * hs_scrub_start starts one thread per context that wakes every period_us microseconds.  Each tick takes the audit's turn (it is
 * serialised with hs_table_audit, hs_table_repair, hs_committee_stage and hs_committee_commit) and audits one slice:
 *   - the next slots_per_tick key slots in service, in slot order and wrapping at the end (the slots out of service between them have
 *     no table and come free): their comb tables, with hs_table_audit's checks;
 *   - the next base_entries_per_tick entries of the base-point table (entry e is entry e % (2^(w-1) + 1) of window e / (2^(w-1) + 1));
 *   - the KEY, FLAG and LOOKUP checks of every slot and every hash entry: a thread each, so every tick runs them all.
 *   A pass is complete when every slot in service and every base entry has been audited since it began; a pass takes
 *   max(ceil(slots in service / slots_per_tick), ceil(base entries / base_entries_per_tick)) ticks, and the next one starts from slot 0
 *   and entry 0.  The kernels run on the audit's private lowest-priority stream; the context's mutex is held only to snapshot and enqueue,
 *   as in hs_table_audit.
 *   - Authority: the map given (expect_pks / expect_live, nullable, n_slots == hs_key_slots) or, with NULL, the engine's host mirror,
 *     with hs_table_audit's rules.  A registration, hs_committee_update, hs_committee_commit or a key-cache change makes it stale: from
 *     then on every tick pauses (and counts the pause) until hs_scrub_set_map gives the map of the new slots.  No tick audits against a
 *     stale map, and a committee change is never reported as a finding.  A pending stage is not a change.  A new map starts a new pass.
 *   - Repair: a tick that finds anything also audits the tables of the slots its slot checks flagged, repairs exactly what it found from
 *     the same authority as hs_table_repair does (failing slots rebuilt and proved off the verify path, the hash table rebuilt, the
 *     base-point table rebuilt with the device drained; every verify queue's signature and certificate caches emptied), then audits its
 *     slice and those slots again.  A slot whose repair fails stays out of service.  Then cb (nullable) runs once, on the scrub's thread:
 *     found = the HS_AUDIT_* classes found, failed = those the second audit still finds (0: all repaired), first_slot = the lowest slot
 *     with a finding ((size_t)-1: only the base-point table or a stray hash entry).  cb may call hs_scrub_set_map and any entry point
 *     but hs_scrub_stop and hs_ctx_destroy.
 *   - HS_ERR_ARG: a scrub already runs on ctx, period_us, slots_per_tick or base_entries_per_tick is 0, or the map breaks the audit's
 *     rules.  A CUDA error in a tick ends the thread; hs_scrub_stop returns it.
 *   - hs_scrub_stop joins the thread (waiting for a tick in progress); a no-op returning HS_OK when none runs.  hs_ctx_destroy calls it.
 *   - hs_scrub_stats: the counters of the current or last scrub, readable at any time.
 *   Without hs_scrub_start nothing of this runs.  A multi-device context is scrubbed member by member (hs_multi_member). */
typedef void(hs_scrub_cb)(void *user, uint32_t found, uint32_t failed, size_t first_slot); /* HS_AUDIT_* bits */
int hs_scrub_start(hs_ctx *ctx, const uint8_t *expect_pks_or_null /* n_slots x 32 */, const uint32_t *expect_live_or_null /* bitmap */,
                   size_t n_slots, uint32_t period_us, uint32_t slots_per_tick, uint32_t base_entries_per_tick, hs_scrub_cb *cb_or_null,
                   void *user);
int hs_scrub_set_map(hs_ctx *ctx, const uint8_t *expect_pks_or_null /* n_slots x 32 */, const uint32_t *expect_live_or_null /* bitmap */,
                     size_t n_slots);
int hs_scrub_stop(hs_ctx *ctx);
/* passes completed, slots audited, base entries audited, ticks, findings (slots, the base-point table and stray hash entries with a
 * finding), slots repaired, failed repairs (findings the second audit still finds), ticks paused on a stale map */
#define HS_SCRUB_STATS 8
int hs_scrub_stats(hs_ctx *ctx, uint64_t out[HS_SCRUB_STATS]);
/* on != 0: a tick whose findings can all be mended (hs_table_mend's rules, with the scrub's map) mends them instead of repairing them;
 * a tick with any other finding repairs, as without it.  The callback's found / failed keep their meaning, and the mend's work counts
 * in hs_table_mend_stats, not in the scrub's repaired slots.  Off on a new context; the setting outlives hs_scrub_stop / hs_scrub_start
 * and takes effect from the next tick.  HS_ERR_ARG: ctx NULL. */
int hs_scrub_mend(hs_ctx *ctx, int on);
/* Attaches q (a queue of ctx) to ctx's scrub: from then on every tick also audits the next buckets_per_tick buckets of q's signature
 * cache with hs_queue_sig_audit, wrapping at the end of the table, whether or not the slot map is paused.  A new table (a resize, or
 * the cache turned off and on) starts again at bucket 0; while the cache is off the slice audits nothing.  q_or_null = NULL detaches.
 *   - A tick that corrected an entry calls cb with HS_AUDIT_SIGCACHE in found (first_slot is (size_t)-1 unless a slot had a finding);
 *     failed never carries it.  hs_queue_sig_audit_stats counts the slices and the passes they complete.
 *   - The attachment outlives hs_scrub_stop / hs_scrub_start; hs_queue_destroy(q) detaches q, after a tick in progress.  Without this
 *     call a scrub launches nothing for any queue.
 *   - HS_ERR_ARG: ctx NULL, q of another context, or buckets_per_tick 0 with q given. */
int hs_scrub_sig_cache(hs_ctx *ctx, hs_queue *q_or_null, uint32_t buckets_per_tick);

/* ---- explanation of a verdict: a table-free re-check that names every check a record fails ------------------------------------
 * A verify call answers 0 for malformed bytes, a small-order key or R, a signature over another message and a false reject by the
 * engine alike.  This call re-checks records by a separate method and reports each check of the decision procedure as its own bit
 * (out_why[i], one byte per record).  Every bit is evaluated on its own; there is no "first failure":
 *   HS_WHY_S_NONCANONICAL  S >= l
 *   HS_WHY_A_INVALID       A does not decompress (dalek's tolerant rules)
 *   HS_WHY_R_INVALID       R does not decompress
 *   HS_WHY_A_SMALL         A decompresses and [8]A is the identity
 *   HS_WHY_R_SMALL         R decompresses and [8]R is the identity
 *   HS_WHY_EQUATION        S, A and R all parse and [S]B + [k](-A) != R as points (cofactorless, k = SHA-512(R || A || msg) mod l);
 *                          clear when any of them does not parse
 * The mask restates both verdicts:  strict verdict 1  <=>  why == 0;
 *                                   batch-eq verdict 1  <=>  (why & ~(HS_WHY_A_SMALL | HS_WHY_R_SMALL)) == 0.
 *   - Use: explain the rejected record of a rejected message (log the mask with it).  A record the verify paths rejected but this call
 *     finds valid in its mode is an engine fault, not a bad signature: audit and repair the tables (hs_table_repair) and answer that
 *     message on another verifier.
 *   - Method: one thread per record computes [S]B and [k](-A) with a radix-16 window on the points themselves (B included), and decides
 *     small order by three doublings.  It reads no context table: no per-key comb table, key slot, key flag or hash table, and not the
 *     base-point table.  So it does not depend on the committee, the table geometry, the key cache, or an audit or repair in progress.
 *     It is slower than a verify and meant for the rare rejected record, not for every record.
 *   - Isolation: it does not teach the key cache and touches no verify queue (ring, caches, counters).  Its launches count in
 *     hs_kernel_launches.  n == 0 returns HS_OK and launches nothing; NULL recs or out_why with n > 0 is HS_ERR_ARG and writes nothing. */
#define HS_WHY_S_NONCANONICAL 1u
#define HS_WHY_A_INVALID 2u
#define HS_WHY_R_INVALID 4u
#define HS_WHY_A_SMALL 8u
#define HS_WHY_R_SMALL 16u
#define HS_WHY_EQUATION 32u
int hs_explain_rec128(hs_ctx *ctx, const hs_rec128 *recs, size_t n, uint8_t *out_why /* n */);

/* ---- device-resident entry points (inputs already in HBM; enqueue on `stream`, a cudaStream_t) -------------------
 * Every kernel and copy of a call is ordered after the caller's earlier work on `stream`; misses of the committee lookup run on an
 * internal stream and join back into `stream` before the finish kernel.  The calls take no mutex (see Conventions): one thread and one
 * stream at a time per context.  A host-pointer call made after a verify pass (rec128, var, committee, msgs, qc_votes, groups) waits
 * on the device for the latest such pass before it reuses the shared scratch; with deferred mode on, host-pointer calls must still not
 * be mixed with deferred passes in flight (hs_set_deferred). */
int hs_verify_rec128_dev(hs_ctx *ctx, const void *d_recs, size_t n, uint32_t mode, void *d_bitmap, void *stream);
int hs_verify_var_dev(hs_ctx *ctx, const void *d_sig, const void *d_pk, const void *d_msgs, const void *d_off, size_t n,
                      uint32_t mode, void *d_bitmap, void *stream);
int hs_verify_committee_dev(hs_ctx *ctx, const void *d_validator_idx, const void *d_sig, const void *d_msg_idx,
                            const void *d_digests, size_t n, uint32_t mode, void *d_bitmap, void *stream);
int hs_digest32_dev(hs_ctx *ctx, const void *d_data, const void *d_off, size_t n, void *d_out, void *stream);
/* Digest of n fixed-size messages (msg_len bytes each, concatenated): the transaction / payload shape.  16-byte aligned sizes
 * >= 128 take the staged kernel (coalesced loads; multiples of 128 also skip the padding block's message schedule). */
int hs_digest32_fixed_dev(hs_ctx *ctx, const void *d_msgs, size_t msg_len, size_t n, void *d_out, void *stream);
/* d_digests: n x 32 bytes of scratch that receives Digest(msg_i). */
int hs_verify_msgs_dev(hs_ctx *ctx, const void *d_sig, const void *d_pk_or_null, const void *d_validator_idx_or_null, const void *d_msgs,
                       size_t msg_len, size_t n, uint32_t mode, void *d_digests, void *d_bitmap, void *stream);

/* QC votes of this rank's shard (per-vote verify_batch condition) over precomputed QC digests (hs_digest32_fixed_dev over the
 * 40-byte preimages), and the per-QC AND over a (possibly all-gathered) vote bitmap — the device-resident pieces of
 * hs_verify_qcs, used when the votes of many QCs are sharded across GPUs (BASELINE config[3]). */
int hs_verify_qc_votes_dev(hs_ctx *ctx, const void *d_qc_digests, const void *d_pk_or_null, const void *d_validator_idx_or_null, const void *d_sig,
                           const void *d_qc_idx, size_t n_votes, void *d_vote_bitmap, void *stream);
/* d_qc_bitmap bit j = AND of the bits of d_vote_bitmap whose d_qc_idx is j (no such bit -> 1), over n_votes bits.  The same AND reduces
 * the item bitmap of hs_verify_groups_dev to group verdicts: pass the items' group indices as d_qc_idx and the group count as n_qc. */
int hs_qc_and_dev(hs_ctx *ctx, const void *d_vote_bitmap, const void *d_qc_idx, size_t n_votes, size_t n_qc, void *d_qc_bitmap, void *stream);

/* hs_verify_groups with every array in device memory, enqueued on `stream`.  Item i is (sig[i], key_i) over
 * Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i]+1])), hashed on the GPU, judged by mode[i] (NULL = all strict).
 * d_item_bitmap bit i = item i's verdict in ITS OWN mode.  Group verdicts: hs_qc_and_dev(d_item_bitmap, d_group_idx, ...).
 *   - Arrays: preimages (bytes), pre_off (uint64, n_msgs + 1), sig (64 B each), pk (32 B each) or validator_idx (uint32; used when pk is
 *     NULL: the committee-indexed form, which needs a registered committee), msg_idx (uint32), mode (uint8), d_item_bitmap (uint32 words).
 *   - Mode bytes: HS_MODE_BATCH_EQ (1) selects the verify_batch condition; ANY other value selects strict (hs_verify_groups, which
 *     runs this pass, rejects bytes > 1 first; this form cannot see them).
 *   - Device arrays are trusted, as in hs_verify_var_dev and hs_digest32_dev: offsets, indices and lengths are not checked.  HS_ERR_ARG
 *     covers only what the host can see: NULL pointers, n_items > 0 with n_msgs == 0, the committee-indexed form without a committee.
 *   - Keys take the paths of every other pass: key bytes are looked up in the committee (misses take the generic kernel), without a
 *     committee the key cache or the generic kernel.  The engine hashes the preimages into its own scratch.
 *   - Deferred mode (hs_set_deferred) and hs_peer_next work as for the other `_dev` verify calls: the finish kernel runs on the tail
 *     stream; an armed call stores its item words into every peer's buffer at word_offset (and n_items == 0 still sends the epoch flag).
 *     sig, pk / validator_idx and mode must stay valid until hs_results_wait. */
int hs_verify_groups_dev(hs_ctx *ctx, const void *d_preimages, const void *d_pre_off /* n_msgs + 1 */, size_t n_msgs, const void *d_sig,
                         const void *d_pk_or_null, const void *d_validator_idx_or_null, const void *d_msg_idx, const void *d_mode_or_null,
                         size_t n_items, void *d_item_bitmap, void *stream);
/* Explanation of the rejected items of a device-resident pass, on the GPU, with nothing copied to the host: the table-free re-check of
 * hs_explain_rec128 for every item whose bit is 0, and a count of engine faults (items rejected that the re-check finds valid in their mode).
 *   - Inputs: the arrays of an hs_verify_groups_dev pass (preimages, pre_off, sig, msg_idx, mode) with KEY BYTES in pk, and d_item_bitmap,
 *     that pass's item bitmap or any bitmap the caller builds.  Item i is examined when its bit is 0: the lowest-index max_explain such
 *     items, or all of them with max_explain = 0.  Selection is by item index, so the result is deterministic.
 *   - d_why[i] (n_items bytes): for an examined item, byte for byte what hs_explain_rec128 returns for the record (sig[i], pk[i],
 *     SHA-512(preimage of msg_idx[i])[..32]); every other byte is HS_WHY_NOT_EXAMINED.
 *   - d_out (HS_EXPLAIN_DEV_OUT uint32 words): [0] items whose bit is 0, [1] items examined, [2] engine faults among them, [3] the lowest
 *     index of an engine fault (0xffffffff: none).  An examined item is an engine fault when its mask is 0 under a strict mode byte (any
 *     byte but 1, or a NULL mode array: hs_verify_groups_dev treats every byte other than 1 as strict), or has no bit other than
 *     HS_WHY_A_SMALL | HS_WHY_R_SMALL under mode byte 1.  A node that sees out[2] > 0 audits and repairs its tables and answers those
 *     messages on another verifier.
 *   - Keys are always key bytes, and the call reads no context table (no comb table, key slot, flag, hash table or base-point table), as
 *     hs_explain_rec128.  For a committee-indexed pass, pass the caller's own index -> key map gathered by validator index (map[vidx]), so
 *     the check does not depend on the tables it is meant to doubt.
 *   - Ordering: enqueued on `stream`, after the caller's earlier work there; the bitmap is read in stream order.  In deferred mode the
 *     stream first waits on the device for the pass tails already enqueued (as hs_results_wait); there is no host wait.
 *   - Scratch: its own, not the verify scratch, so host-pointer calls do not wait for it.  Growing it (the first call, or a larger one)
 *     may synchronise the device, as other `_dev` scratch growth does.  The re-check runs on at most a quarter of the SMs (the explain
 *     lane's share), grid-stride beyond that, so a flood of junk leaves the other SMs to verify work on other streams.
 *   - Isolation: it does not teach the key cache and touches no verify queue, cache or counter; its launches count in hs_kernel_launches.
 *   - n_items == 0 returns HS_OK, writes nothing and launches nothing.  HS_ERR_ARG writes nothing: NULL required pointers (all but
 *     mode) or n_msgs == 0 with n_items > 0, or n_items above 2^32 - 1.  Device arrays are trusted, as in hs_verify_groups_dev. */
#define HS_WHY_NOT_EXAMINED 0x80u /* this call only: the item was accepted, or is past max_explain */
#define HS_EXPLAIN_DEV_OUT 4
int hs_explain_groups_dev(hs_ctx *ctx, const void *d_preimages, const void *d_pre_off /* n_msgs + 1 */, size_t n_msgs, const void *d_sig,
                          const void *d_pk, const void *d_msg_idx, const void *d_mode_or_null, const void *d_item_bitmap, size_t n_items,
                          size_t max_explain, void *d_why /* n_items bytes */, void *d_out /* HS_EXPLAIN_DEV_OUT x uint32 */, void *stream);

/* ---- load generation: RFC 8032 key generation and signing of 32-byte digests ON THE GPU ---------------------------------------
 * generate_keypair / Signature::new (crypto/src/lib.rs:167-175,185-191) for input synthesis only: the node itself signs one
 * message per request on the CPU (SignatureService) and keeps doing so.  Deterministic, byte-identical to dalek / OpenSSL.
 * Signature i is over digests[i] with key key_idx[i] (NULL: key i).  Secret seeds travel to the device: test / benchmark use. */
int hs_keygen_batch(hs_ctx *ctx, const uint8_t *seeds /* n x 32 */, size_t n, uint8_t *out_pks /* n x 32 */);
int hs_sign_digests(hs_ctx *ctx, const uint8_t *seeds, const uint8_t *pks, size_t n_keys, const uint32_t *key_idx_or_null,
                    const uint8_t *digests /* n x 32 */, size_t n, uint8_t *out_sig /* n x 64 */);
int hs_keygen_batch_dev(hs_ctx *ctx, const void *d_seeds, size_t n, void *d_pks, void *stream);
int hs_sign_digests_dev(hs_ctx *ctx, const void *d_seeds, const void *d_pks, size_t n_keys, const void *d_key_idx_or_null, const void *d_digests,
                        size_t n, void *d_sig, void *stream);

/* Deferred-results mode for STREAMS of `_dev` verify passes (e.g. one pass per QC burst): the latency-bound tail of a pass — finish
 * kernel incl. the peer exchange, hs_qc_and_dev — runs on an internal stream and overlaps the main kernel of the next pass (a serial
 * field inversion per block makes the tail ~80 us however small the pass).  Bitmaps are complete only after hs_results_wait(ctx, stream),
 * which makes `stream` wait for every tail enqueued so far; the signatures of a pass must stay valid until then.  Host-pointer entry points
 * must not be mixed with deferred passes in flight. */
int hs_set_deferred(hs_ctx *ctx, int on);
int hs_results_wait(hs_ctx *ctx, void *stream);

/* ---- multi-GPU: fused all-gather of the accept bitmap (one process per GPU, same node, NVLink) ------------------------
 * Each rank creates a result buffer for the GLOBAL bitmap (total_words) and exports a 64-byte CUDA-IPC handle; the host
 * exchanges handles (e.g. torch.distributed.all_gather_object) and opens every peer's.  hs_peer_next() then arms the next
 * `_dev` verify call: its finish kernel stores each bitmap word it produces directly into EVERY rank's buffer at
 * word_offset (P2P stores over NVLink), signals the peers and waits for theirs — after the call (stream order) the buffer
 * returned by hs_peer_bitmap() holds every rank's verdicts for that epoch.  Epochs must increase by one per armed call.
 * The buffer is double-buffered by epoch parity (hs_peer_bitmap() follows the most recently armed epoch): consume epoch e's
 * bitmap on the same stream before enqueueing the verify of epoch e+1 and no barrier between ranks is needed.  The flag
 * exchange runs inside the finish kernel (no extra launches).  total_words must be world x (words per rank); a peer that
 * never signals makes hs_peer_timed_out() return 1 and its shard read as all-rejected.  hs_peer_setup may be called again
 * (new total_words): the old buffers are released — every rank must have drained its stream and re-exchange handles. */
int hs_peer_setup(hs_ctx *ctx, int rank, int world, size_t total_words, uint8_t handle_out[64]);
int hs_peer_open(hs_ctx *ctx, int peer_rank, const uint8_t handle[64]);
int hs_peer_next(hs_ctx *ctx, size_t word_offset, uint32_t epoch);
void *hs_peer_bitmap(hs_ctx *ctx);
int hs_peer_timed_out(hs_ctx *ctx);

/* ---- several GPUs in one process: a multi-device context that shards the host-pointer verify calls ------------------------------
 * A node is one process (its Core task and its mempool Processors call `crypto` from it), so it cannot reach a second GPU through the
 * one-process-per-GPU route above.  A multi-device context is n_devices ordinary contexts, its MEMBERS, plus host code that splits a call
 * across them.
 *   - Verdicts: every output is bit for bit what the same single-context call returns, with or without a registered committee, in both
 *     modes and with mixed mode bytes.  Members may run different table geometries (each picks its per-key window from its own free memory
 *     and budget); verdicts do not depend on geometry.
 *   - Sharding: a call is sharded only when every member gets at least HS_MULTI_MIN_SHARD records.  Member i then verifies a contiguous
 *     record range; every range but the last starts at a multiple of 32 records, so each member writes whole words of the caller's bitmap.
 *     hs_multi_verify_groups gives each member its item range with the whole preimage arrays and n_groups; each member ANDs its items into
 *     group words of its own (a group with no item in its range stays 1) and the caller's group words are the AND of the members' words.
 *   - A smaller call runs whole on one member, chosen round-robin, without the multi-context's lock: small calls from several threads run
 *     on different GPUs at once, and calls of up to 64 records keep the one-launch latency path.
 *   - Threads and locks: hs_multi_create starts one worker thread per member after the first; the calling thread runs member 0's range.
 *     Sharded calls and committee changes are serialised on the multi-context's mutex, and each member still serialises on its own, so a
 *     verify queue created on a member (hs_multi_member) keeps working beside them.  A device may be listed more than once.
 *   - Errors: the argument checks of hs_verify_rec128 / hs_verify_msgs / hs_verify_groups cover the whole call before any member runs, so
 *     HS_ERR_ARG writes nothing.  A member's failure returns that member's status and hs_multi_last_error names the member (index, device)
 *     with its hs_last_error; the outputs are then undefined and the caller rejects every signature of the call.
 *   - Committee: hs_multi_committee_register registers on every member at once.  If any member fails, or the members' out_valid_bitmap
 *     differ (HS_ERR_CUDA), every member ends with NO committee.  hs_multi_committee_update must give every member the same out_add_idx;
 *     a mismatch is HS_ERR_CUDA, and after any failure of it the members may differ: re-register.  A staged change
 *     (hs_committee_stage / _commit / _discard) is made member by member through hs_multi_member with the same arguments, as a repair is:
 *     stage on every member (at once, from one thread per member); if any stage fails or the members return different indices, discard
 *     on every member; otherwise commit on every member.  After a failed commit the members may differ: re-register.  The bindings do
 *     exactly this (MultiEngine.stage_committee / commit_committee / discard_committee, hs::MultiEngine, multi::Multi).  A staged
 *     registration (hs_committee_stage_register) is made the same way, and is committed only when every member staged with the same
 *     out_valid_bitmap and window: a failed or mismatched stage is discarded on every member, which all keep their committee
 *     (MultiEngine.stage_register_committee, hs::MultiEngine::stage_register_committee, multi::Multi::stage_register_committee).  Apart from that,
 *     the committee-indexed forms need every member's committee changed through the two calls above: never change one member alone.
 *   - Pinned memory from hs_host_alloc (cudaMallocHost) is portable under UVA: every member DMAs from the caller's pinned buffers directly.
 *   - hs_multi_destroy joins the workers and destroys the members (and the verify queues created on them); it must not race with calls.
 *     A failed hs_multi_create (n_devices == 0, a bad ordinal, no memory) leaves no thread and no member behind. */
#define HS_MULTI_MIN_SHARD 4096 /* records per member below which a call runs whole on one member */
typedef struct hs_multi hs_multi;
/* flags as hs_ctx_create, applied to every member. */
int hs_multi_create(hs_multi **out, const int *devices, size_t n_devices, uint32_t flags);
void hs_multi_destroy(hs_multi *m);
/* The last failure on this multi-context (never NULL): a member's failure names the member (index, device) and its hs_last_error. */
const char *hs_multi_last_error(const hs_multi *m);
size_t hs_multi_members(const hs_multi *m);
/* Member i (borrowed; NULL when out of range): every single-device entry point works on it. */
hs_ctx *hs_multi_member(hs_multi *m, size_t i);
int hs_multi_committee_register(hs_multi *m, const uint8_t *pks /* N x 32 */, size_t N, uint32_t *out_valid_bitmap);
int hs_multi_committee_update(hs_multi *m, const uint8_t *add_pks /* n_add x 32 */, size_t n_add, const uint32_t *remove_idx, size_t n_remove,
                              uint32_t *out_add_idx);
/* The arguments and outputs of hs_verify_rec128, hs_verify_msgs and hs_verify_groups. */
int hs_multi_verify_rec128(hs_multi *m, const hs_rec128 *recs, size_t n, uint32_t mode, uint32_t *out_bitmap);
int hs_multi_verify_msgs(hs_multi *m, const uint8_t *sig /* n x 64 */, const uint8_t *pk_or_null /* n x 32 */, const uint32_t *validator_idx_or_null,
                         const uint8_t *msgs, size_t msg_len, size_t n, uint32_t mode, uint32_t *out_bitmap);
int hs_multi_verify_groups(hs_multi *m, const uint8_t *preimages, const uint64_t *pre_off /* n_msgs + 1 */, size_t n_msgs,
                           const uint8_t *sig /* n_items x 64 */, const uint8_t *pk_or_null, const uint32_t *validator_idx_or_null,
                           const uint32_t *msg_idx, const uint32_t *group_idx, const uint8_t *mode_or_null, size_t n_items, size_t n_groups,
                           uint32_t *out_item_bitmap_or_null, uint32_t *out_group_bitmap);

#ifdef __cplusplus
}
#endif
#endif
