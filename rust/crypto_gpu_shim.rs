// crypto/src/gpu.rs — FFI to libhs_crypto.so (include/hs_crypto.h) for asonnino/hotstuff's `crypto` crate.
//
// STATUS: source only — this image has no cargo/rustc, so this file has never been compiled here.  The same C ABI is exercised
// end to end by tests/ (ctypes) and tests/cpp/crypto_tests.cpp.  INTEGRATION.md §2 shows the edits in crypto/src/lib.rs.
//
// What it adds over a bare FFI pass-through:
//   * CPU/GPU cut-over (SURVEY §8f.2): a lone signature or a single large Digest stays on the reference's own dalek / sha2 path;
//     the GPU takes every call with >= GPU_MIN_SIGS signatures and every multi-message digest.  One verify costs the
//     GPU about what one CPU core needs (a square-root chain in a lone warp), a few votes are already cheaper on the GPU, and one
//     large digest is a sequential SHA-512 chain that a CPU core runs faster; tools/replay_config5 measures the three calls.
//   * every status code is propagated: a failed registration or engine call is an Err / a rejected message, never an accept.
//   * batch front ends for the consensus call sites: many QCs (view-change burst), TC votes, and whole bincode frames
//     (ingest_frames + verify_ingested: the receiver path of consensus.rs:138 without building the message structs first).
use std::os::raw::c_int;
use std::sync::atomic::{AtomicBool, Ordering};
use std::sync::{Mutex, OnceLock};

/// The verify queue (hs_queue_*): concurrent single-message verifies share latency-path launches (`queue::verify_queued`).
#[path = "crypto_gpu_queue.rs"]
pub mod queue;
/// Whole certificates through the same queue (hs_queue_submit_group): Block / Timeout / TC verifies at the connection tasks
/// (`group_queue::verify_group_queued`).
#[path = "crypto_gpu_group_queue.rs"]
pub mod group_queue;
/// The same with the signed preimages instead of their Digests (hs_queue_submit_msgs): the GPU hashes them, so a TC's votes cost
/// the connection task no SHA-512 calls (`msgs_queue::verify_msgs_queued`).
#[path = "crypto_gpu_msgs_queue.rs"]
pub mod msgs_queue;
/// The queue's certificate cache (hs_queue_cert_cache): a QC that several Timeouts carry is verified once
/// (`msgs_queue::verify_timeout_queued`).
#[path = "crypto_gpu_cert_cache.rs"]
pub mod cert_cache;
/// The queue's signature cache (hs_queue_sig_cache): a vote verified in a Timeout is a cache hit in the TC and the Block after
/// it.  Turned on with the certificate cache (`cert_cache::enable`).
#[path = "crypto_gpu_sig_cache.rs"]
pub mod sig_cache;
/// Sharing of that cache (hs_queue_sig_share) with the synchronous fallbacks for TCs and Blocks above GROUP_MAX_SIGS and with the
/// batch lane: the votes the queue verified in the Timeouts are hits there too.  Turned on with the cache (`sig_cache::enable`).
#[path = "crypto_gpu_sig_share.rs"]
pub mod sig_share;
/// The audit of that cache (hs_queue_sig_audit): every held entry re-checked from its bytes and a wrong flag byte corrected, a slice
/// per scrub tick (`sig_audit::attach`) and the whole table on an `engine_fault` (`sig_audit::audit_cache`).
#[path = "crypto_gpu_sig_audit.rs"]
pub mod sig_audit;
/// The queue's generic-key device path (hs_queue_generic): a request with a key outside the registered committee is verified by a
/// queue kernel instead of holding up the queue's thread.  Turned on when the node-wide queue is created (`queue::queue`).
#[path = "crypto_gpu_generic_queue.rs"]
pub mod generic_queue;
/// The queue's batch lane (hs_queue_submit_batch): a whole hs_verify_groups pass (a large Block, a collected view-change burst)
/// awaited by a task instead of run under `spawn_blocking` (`batch_queue::verify_groups_queued`).
#[path = "crypto_gpu_batch_queue.rs"]
pub mod batch_queue;
/// The queue's explain lane (hs_queue_submit_explain): every rejected record of a rejected message explained in one non-blocking
/// request, without holding the context's mutex for the re-check (`explain_queue::explain_rejected_queued`).
#[path = "crypto_gpu_explain_queue.rs"]
pub mod explain_queue;
/// The device-resident certificate pass (hs_verify_groups_dev): Blocks, Timeouts and TCs whose arrays are already in HBM, enqueued on
/// the caller's stream (`groups_dev::verify_groups_dev`).
#[path = "crypto_gpu_groups_dev.rs"]
pub mod groups_dev;
/// The explanation of such a pass's rejected items on the GPU (hs_explain_groups_dev): a why byte per rejected item and a count of
/// engine faults, with nothing copied to the host (`explain_dev::explain_rejected_dev`).
#[path = "crypto_gpu_explain_dev.rs"]
pub mod explain_dev;
/// Several GPUs from this one process (hs_multi_*): large verifies sharded across them, small ones spread round-robin
/// (`multi::Multi`).
#[path = "crypto_gpu_multi.rs"]
pub mod multi;
/// The engine-owned scrub of the live key tables (hs_scrub_*): a bounded slice audited and repaired per tick against the node's map,
/// started once after `self_test` (`scrub::start`) and given the new map after every committee change.
#[path = "crypto_gpu_scrub.rs"]
pub mod scrub;
/// The mend of corrupt comb-table entries in place (hs_table_mend*, hs_scrub_mend): what the audit finds fixed with no drain and no
/// validator out of service, with `audit_tables` (the repair) for what it leaves (`mend::mend_tables`, `mend::attach_scrub`).
#[path = "crypto_gpu_mend.rs"]
pub mod mend;
/// The staged registration (hs_committee_stage_register): the next committee's whole key store built and proved beside the live one,
/// switched in at the boundary with one drain, for a change the spare slots cannot hold or a new window (`stage_register_committee`,
/// `commit_registration`).
#[path = "crypto_gpu_stage_register.rs"]
pub mod stage_register;
pub use stage_register::{commit_registration, discard_registration, stage_register_committee};

#[repr(C)] pub struct HsCtx { _private: [u8; 0] }
#[repr(C)] #[derive(Clone, Copy)] pub struct HsRec128 { pub sig: [u8; 64], pub pk: [u8; 32], pub msg: [u8; 32] } // (Signature, PublicKey, Digest)
#[repr(C)] #[derive(Clone, Copy)] pub struct HsVote   { pub pk: [u8; 32], pub sig: [u8; 64] }                     // QC.votes element, messages.rs:168

/// Mirror of hs_frame_info (48 bytes): which items of the ingest output belong to frame i's author signature / QC votes / TC votes.
#[repr(C)] #[derive(Clone, Copy, Default)]
pub struct HsFrameInfo { pub kind: u8, pub has_tc: u8, pub qc_is_genesis: u8, pub pad: u8, pub author_item: u32,
                         pub qc_lo: u32, pub qc_hi: u32, pub tc_lo: u32, pub tc_hi: u32, pub round: u64, pub qc_round: u64, pub tc_round: u64 }
/// Mirror of hs_ingest_out: caller-owned arrays (capacities in, counts out).
#[repr(C)]
pub struct HsIngestOut { pub cap_items: usize, pub cap_msgs: usize, pub cap_pre_bytes: usize,
                         pub sig: *mut u8, pub pk: *mut u8, pub msg_idx: *mut u32, pub group_idx: *mut u32, pub mode: *mut u8,
                         pub preimages: *mut u8, pub pre_off: *mut u64, pub n_items: usize, pub n_msgs: usize, pub pre_bytes: usize }
pub const HS_FRAME_MALFORMED: u8 = 255;

pub const HS_OK: c_int = 0;
pub const HS_ERR_ARG: c_int = 2;
pub const HS_ERR_NOMEM: c_int = 3;
pub const HS_ERR_SELFTEST: c_int = 4;
/// Verdict mode bytes (HS_MODE_*): 0 = Signature::verify (strict), 1 = the per-signature condition of Signature::verify_batch.
pub const HS_MODE_BATCH_EQ: u8 = 1;
/// hs_explain_rec128's bits, one per check a record fails: S >= l, A / R do not decompress, A / R of small order, the equation.
pub const HS_WHY_S_NONCANONICAL: u8 = 1;
pub const HS_WHY_A_INVALID: u8 = 2;
pub const HS_WHY_R_INVALID: u8 = 4;
pub const HS_WHY_A_SMALL: u8 = 8;
pub const HS_WHY_R_SMALL: u8 = 16;
pub const HS_WHY_EQUATION: u8 = 32;
/// Smallest signature count sent to the GPU (below it the dalek path is faster on this hardware; see the header comment).
pub const GPU_MIN_SIGS: usize = 2;
/// A Digest call goes to the GPU only with at least this many messages in flight (SHA-512 is sequential inside one message).
pub const GPU_MIN_DIGEST_MSGS: usize = 8;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_ctx_create(out: *mut *mut HsCtx, device: c_int, flags: u32) -> c_int;
    fn hs_last_error(ctx: *const HsCtx) -> *const std::os::raw::c_char;
    fn hs_committee_register(ctx: *mut HsCtx, pks: *const u8, n: usize, out_valid_bitmap: *mut u32) -> c_int;
    fn hs_committee_update(ctx: *mut HsCtx, add_pks: *const u8, n_add: usize, remove_idx: *const u32, n_remove: usize, out_add_idx: *mut u32) -> c_int;
    fn hs_committee_stage(ctx: *mut HsCtx, add_pks: *const u8, n_add: usize, remove_idx: *const u32, n_remove: usize, out_add_idx: *mut u32) -> c_int;
    fn hs_committee_commit(ctx: *mut HsCtx) -> c_int;
    fn hs_committee_discard(ctx: *mut HsCtx) -> c_int;
    fn hs_verify_strict_batch(ctx: *mut HsCtx, recs: *const HsRec128, n: usize, out_bitmap: *mut u32) -> c_int;
    fn hs_verify_batch_shared_msg(ctx: *mut HsCtx, digest: *const u8, votes: *const HsVote, n: usize,
                                  all_ok: *mut c_int, out_bitmap_or_null: *mut u32) -> c_int;
    fn hs_verify_qcs(ctx: *mut HsCtx, preimages: *const u8, n_qc: usize, pk: *const u8, vidx: *const u32, sig: *const u8,
                     qc_idx: *const u32, n_votes: usize, out_vote_bitmap: *mut u32, out_qc_bitmap: *mut u32) -> c_int;
    fn hs_verify_tcs(ctx: *mut HsCtx, tc_rounds: *const u64, n_tc: usize, pk: *const u8, vidx: *const u32, sig: *const u8,
                     high_qc_rounds: *const u64, tc_idx: *const u32, n_votes: usize, out_vote_bitmap: *mut u32, out_tc_bitmap: *mut u32) -> c_int;
    fn hs_digest32_batch(ctx: *mut HsCtx, data: *const u8, off: *const u64, n: usize, out: *mut u8) -> c_int;
    fn hs_verify_groups(ctx: *mut HsCtx, preimages: *const u8, pre_off: *const u64, n_msgs: usize, sig: *const u8, pk: *const u8, vidx: *const u32,
                        msg_idx: *const u32, group_idx: *const u32, mode: *const u8, n_items: usize, n_groups: usize,
                        out_item_bitmap: *mut u32, out_group_bitmap: *mut u32) -> c_int;
    fn hs_ingest_consensus_frames(frames: *const u8, off: *const u64, n: usize, info: *mut HsFrameInfo, out: *mut HsIngestOut) -> c_int;
    fn hs_self_test(ctx: *mut HsCtx, key_bits: c_int, recs: *const HsRec128, expect: *const u8, n: usize, out_failed_paths: *mut u32) -> c_int;
    fn hs_table_audit(ctx: *mut HsCtx, expect_pks: *const u8, expect_live: *const u32, n_slots: usize, out_slot_bits: *mut u8, out_failed: *mut u32) -> c_int;
    fn hs_table_repair(ctx: *mut HsCtx, expect_pks: *const u8, expect_live: *const u32, n_slots: usize, out_slot_bits: *mut u8, out_found: *mut u32,
                       out_failed: *mut u32) -> c_int;
    fn hs_explain_rec128(ctx: *mut HsCtx, recs: *const HsRec128, n: usize, out_why: *mut u8) -> c_int;
}

struct Ctx(*mut HsCtx);
unsafe impl Send for Ctx {}
unsafe impl Sync for Ctx {}            // host-pointer entry points are serialised on the context's mutex
static CTX: OnceLock<Option<Ctx>> = OnceLock::new();
/// Set when `self_test` fails: the engine gives wrong answers on this box, so every call below answers None (the dalek path).
static DISABLED: AtomicBool = AtomicBool::new(false);
/// The node-side index -> key map of the registered committee (None = a freed index): registration order, then every update's
/// removals and returned indices.  `audit_tables` checks the engine's slots against it after every change.
static KEYS: Mutex<Vec<Option<[u8; 32]>>> = Mutex::new(Vec::new());
/// What the engine holds staged, mirrored here: it has one stage, of either kind, and hs_committee_commit / hs_committee_discard apply
/// to whichever is pending.  A change (`stage_committee`) is applied to KEYS by `commit_committee`: the added keys, their indices and the
/// removed indices (KEYS lists no staged index before the commit: the engine holds staged slots out of service, and the audit would
/// report one).  A registration (`stage_register::stage_register_committee`) replaces KEYS at `stage_register::commit_registration`.
/// Each commit and discard checks the kind before it calls the engine; a registration or update clears it, as the engine does.
enum Staged {
    Change { add: Vec<[u8; 32]>, idx: Vec<u32>, remove: Vec<u32> },
    Registration(Vec<[u8; 32]>),
}
static STAGED: Mutex<Option<Staged>> = Mutex::new(None);

/// None when no GPU / the library failed to initialise / the self-test failed: every caller below then stays on the CPU path.
fn ctx() -> Option<*mut HsCtx> {
    if DISABLED.load(Ordering::Acquire) { return None; }
    CTX.get_or_init(|| {
        let mut p = std::ptr::null_mut();
        if unsafe { hs_ctx_create(&mut p, 0, 0) } == HS_OK && !p.is_null() { Some(Ctx(p)) } else { None }
    }).as_ref().map(|c| c.0)
}
fn last_error(c: *mut HsCtx) -> String {
    unsafe { std::ffi::CStr::from_ptr(hs_last_error(c)).to_string_lossy().into_owned() }
}

#[derive(Debug)]
pub enum GpuError { Unavailable, Engine(String), InvalidKeys(Vec<usize>) }

/// Once per epoch from node/src/node.rs after the committee file is read (consensus/src/config.rs:28-60).  Keys that do not
/// decompress are reported (PublicKey::from_bytes would fail on them at first use, crypto/src/lib.rs:202).
pub fn register_committee(keys: &[[u8; 32]]) -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut valid = vec![0u32; (keys.len() + 31) / 32];
    let rc = unsafe { hs_committee_register(c, keys.as_ptr() as *const u8, keys.len(), valid.as_mut_ptr()) };
    if rc != HS_OK {
        KEYS.lock().unwrap().clear();
        *STAGED.lock().unwrap() = None;  // past its argument checks, a registration discards the engine's stage even when it fails
        return Err(GpuError::Engine(last_error(c)));
    }
    let mut map = KEYS.lock().unwrap();
    *map = keys.iter().map(|k| Some(*k)).collect();
    scrub::set_map(c, &map)?;
    *STAGED.lock().unwrap() = None;  // a registration discards a staged change or registration
    let bad: Vec<usize> = (0..keys.len()).filter(|i| valid[i / 32] >> (i % 32) & 1 == 0).collect();
    if bad.is_empty() { Ok(()) } else { Err(GpuError::InvalidKeys(bad)) }
}
/// Known-answer self-test of every GPU path at the context's table geometry (hs_self_test, built-in vectors, the window in use).  Call
/// it once at start-up, after `register_committee`.  On any failure the GPU is switched off for the life of the process: every call
/// below then returns None and the caller takes its dalek / sha2 path.
pub fn self_test() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut failed = 0u32;
    let rc = unsafe { hs_self_test(c, 0, std::ptr::null(), std::ptr::null(), 0, &mut failed) };
    if rc == HS_OK && failed == 0 { return audit_tables(&KEYS.lock().unwrap()); }
    DISABLED.store(true, Ordering::Release);
    Err(GpuError::Engine(format!("self-test failed (status {}, paths {:#x}): {}", rc, failed, last_error(c))))
}
/// Audit of the live key tables (hs_table_audit): every comb-table entry, key slot and lookup entry of the engine against `expected`,
/// the node's index -> key map (None = a freed index).  `self_test` and `update_committee` call it; between those, `scrub::start`
/// keeps auditing on the engine's own thread.  A finding is repaired once from the same map (hs_table_repair: only the failing slots, lookup
/// entries or base-point table are rebuilt, and the caches of verified records are emptied); the GPU stays on when the repair's own
/// final audit is clean, and is switched off for the life of the process, as after a failed self-test, only when the repair fails.
/// Tables that changed while it ran (a committee change from another task) are audited again.
pub fn audit_tables(expected: &[Option<[u8; 32]>]) -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let pks: Vec<u8> = expected.iter().flat_map(|k| k.unwrap_or([0u8; 32])).collect();
    let mut live = vec![0u32; (expected.len() + 31) / 32];
    for (i, k) in expected.iter().enumerate() { if k.is_some() { live[i / 32] |= 1 << (i % 32); } }
    let mut failed = 0u32;
    let mut rc = HS_OK;
    for _ in 0..3 {
        rc = unsafe { hs_table_audit(c, if expected.is_empty() { std::ptr::null() } else { pks.as_ptr() }, live.as_ptr(), expected.len(),
                                     std::ptr::null_mut(), &mut failed) };
        if !(rc == HS_ERR_ARG && last_error(c).contains("changed during the audit")) { break; }
    }
    if rc == HS_OK && failed == 0 { return Ok(()); }
    if rc == HS_ERR_SELFTEST {
        let mut found = 0u32;
        rc = unsafe { hs_table_repair(c, if expected.is_empty() { std::ptr::null() } else { pks.as_ptr() }, live.as_ptr(), expected.len(),
                                      std::ptr::null_mut(), &mut found, &mut failed) };
        if rc == HS_OK { return Ok(()); }
    }
    DISABLED.store(true, Ordering::Release);
    Err(GpuError::Engine(format!("table audit failed (status {}, classes {:#x}): {}", rc, failed, last_error(c))))
}
/// Why one rejected message was rejected: its first rejected record, that record's HS_WHY_* mask, and whether the engine's verdict
/// disagrees with the mask (`engine_fault`: the engine rejected a record that the table-free re-check finds valid in its mode).
#[derive(Debug, Clone, Copy)]
pub struct Explained { pub index: usize, pub why: u8, pub engine_fault: bool }
/// Explains a rejected message: `recs` are its records, `modes` their verdict modes (HS_MODE_*) and `verdicts` the bits the engine
/// returned for them.  Only the first rejected record is re-checked (hs_explain_rec128, a table-free re-check on the GPU), so a flood of
/// junk signatures costs one extra record per rejected message, not one per signature.  On `engine_fault` the caller audits and repairs
/// the tables (`audit_tables`), re-checks the signature cache (`sig_audit::audit_cache`) and answers that message on the dalek path.  None = no record was rejected, no GPU, or the re-check
/// failed (keep the rejection).
pub fn explain_rejected(recs: &[HsRec128], modes: &[u8], verdicts: &[bool]) -> Option<Explained> {
    let index = verdicts.iter().position(|ok| !ok)?;
    let c = ctx()?;
    let mut why = 0u8;
    let rc = unsafe { hs_explain_rec128(c, &recs[index], 1, &mut why) };
    if rc != HS_OK { return None; }
    let valid = if modes[index] == HS_MODE_BATCH_EQ { why & !(HS_WHY_A_SMALL | HS_WHY_R_SMALL) == 0 } else { why == 0 };
    Some(Explained { index, why, engine_fault: valid })
}
/// Incremental epoch change: returns the table indices of the added validators.
pub fn update_committee(add: &[[u8; 32]], remove_idx: &[u32]) -> Result<Vec<u32>, GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut out = vec![0u32; add.len().max(1)];
    let mut keys = KEYS.lock().unwrap();  // held across the update and its audit: the map and the engine change together
    let rc = unsafe { hs_committee_update(c, add.as_ptr() as *const u8, add.len(), remove_idx.as_ptr(), remove_idx.len(), out.as_mut_ptr()) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    *STAGED.lock().unwrap() = None;  // an update discards a staged change or registration
    out.truncate(add.len());
    for &i in remove_idx { keys[i as usize] = None; }
    for (k, &i) in add.iter().zip(out.iter()) {
        if i as usize >= keys.len() { keys.resize(i as usize + 1, None); }
        keys[i as usize] = Some(*k);
    }
    audit_tables(&keys)?;
    scrub::set_map(c, &keys)?;
    Ok(out)
}
/// hs_committee_stage / hs_committee_commit / hs_committee_discard on one context: the shim's own and, one per member, `multi::Multi`'s.
fn stage_on(c: *mut HsCtx, add: &[[u8; 32]], remove_idx: &[u32]) -> Result<Vec<u32>, GpuError> {
    let mut out = vec![0u32; add.len().max(1)];
    let rc = unsafe { hs_committee_stage(c, add.as_ptr() as *const u8, add.len(), remove_idx.as_ptr(), remove_idx.len(), out.as_mut_ptr()) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    out.truncate(add.len());
    Ok(out)
}
fn commit_on(c: *mut HsCtx) -> Result<(), GpuError> {
    let rc = unsafe { hs_committee_commit(c) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    Ok(())
}
fn discard_on(c: *mut HsCtx) -> Result<(), GpuError> {
    let rc = unsafe { hs_committee_discard(c) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    Ok(())
}
/// Prepares the next epoch's committee while this one verifies (hs_committee_stage): the added validators' tables are built and
/// proved on the GPU's lowest-priority stream, and nothing changes for verification until `commit_committee`.  Returns the indices the
/// added validators will have.  Blocks for the build (about 0.1 ms per key): call it from `spawn_blocking` during the last rounds of
/// the epoch.  An Err naming too few free and spare slots (HS_ERR_NOMEM) means: call `update_committee` at the boundary instead.
pub fn stage_committee(add: &[[u8; 32]], remove_idx: &[u32]) -> Result<Vec<u32>, GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut staged = STAGED.lock().unwrap();
    let idx = stage_on(c, add, remove_idx)?;
    *staged = Some(Staged::Change { add: add.to_vec(), idx: idx.clone(), remove: remove_idx.to_vec() });
    Ok(idx)
}
/// Switches the staged committee in at the epoch boundary (hs_committee_commit: no table is built), applies the change to the node's
/// map as `update_committee` would (additions, then removals) and audits the tables against it.  A staged registration is committed by
/// `stage_register::commit_registration` instead.  If the engine's commit fails, the stage stays recorded: discard it.
pub fn commit_committee() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut keys = KEYS.lock().unwrap();  // held across the commit and its audit: the map and the engine change together
    let mut staged = STAGED.lock().unwrap();
    let (add, idx, remove) = match staged.as_ref() {
        Some(Staged::Change { add, idx, remove }) => (add.clone(), idx.clone(), remove.clone()),
        Some(Staged::Registration(_)) => return Err(GpuError::Engine("commit_committee: a registration is staged (commit_registration)".into())),
        None => return Err(GpuError::Engine("commit_committee: nothing staged".into())),
    };
    commit_on(c)?;
    *staged = None;
    for (k, &i) in add.iter().zip(idx.iter()) {
        if i as usize >= keys.len() { keys.resize(i as usize + 1, None); }
        keys[i as usize] = Some(*k);
    }
    for &i in &remove { keys[i as usize] = None; }
    audit_tables(&keys)?;
    scrub::set_map(c, &keys)
}
/// Drops a staged committee change (hs_committee_discard).  A staged registration is dropped by `stage_register::discard_registration`.
pub fn discard_committee() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut staged = STAGED.lock().unwrap();
    if let Some(Staged::Registration(_)) = *staged {
        return Err(GpuError::Engine("discard_committee: a registration is staged (discard_registration)".into()));
    }
    discard_on(c)?;
    *staged = None;
    Ok(())
}

/// Signature::verify for n triples.  None = "use the CPU path" (no GPU, or too few signatures to pay for a launch);
/// Some(bits) = verdicts.  An engine failure rejects everything (core.rs:434-439 drops a message on any Err).
pub fn verify_strict_many(recs: &[HsRec128]) -> Option<Vec<bool>> {
    if recs.len() < GPU_MIN_SIGS { return None; }
    let c = ctx()?;
    let mut bm = vec![0u32; (recs.len() + 31) / 32];
    let rc = unsafe { hs_verify_strict_batch(c, recs.as_ptr(), recs.len(), bm.as_mut_ptr()) };
    Some((0..recs.len()).map(|i| rc == HS_OK && bm[i / 32] >> (i % 32) & 1 == 1).collect())
}
/// Signature::verify_batch (one digest, n votes).  None = use dalek.
pub fn verify_batch(digest: &[u8; 32], votes: &[HsVote]) -> Option<bool> {
    if votes.len() < GPU_MIN_SIGS { return None; }
    let c = ctx()?;
    let mut ok: c_int = 0;
    let rc = unsafe { hs_verify_batch_shared_msg(c, digest.as_ptr(), votes.as_ptr(), votes.len(), &mut ok, std::ptr::null_mut()) };
    Some(rc == HS_OK && ok == 1)
}
/// QC::verify for many certificates at once (the view-change burst: every Timeout carries a high_qc, core.rs:227).
/// `preimages[j]` = hash || round_le (40 bytes); vote i = (pk[i], sig[i]) of certificate qc_idx[i].  Stake / duplicate checks stay
/// with the caller (messages.rs:182-194).
pub fn verify_qcs(preimages: &[[u8; 40]], pk: &[[u8; 32]], sig: &[[u8; 64]], qc_idx: &[u32]) -> Option<Vec<bool>> {
    let c = ctx()?;
    let mut qbm = vec![0u32; (preimages.len() + 31) / 32 + 1];
    let rc = unsafe { hs_verify_qcs(c, preimages.as_ptr() as *const u8, preimages.len(), pk.as_ptr() as *const u8, std::ptr::null(),
                                    sig.as_ptr() as *const u8, qc_idx.as_ptr(), sig.len(), std::ptr::null_mut(), qbm.as_mut_ptr()) };
    Some((0..preimages.len()).map(|j| rc == HS_OK && qbm[j / 32] >> (j % 32) & 1 == 1).collect())
}
/// TC::verify (tc_idx = Some) / n Timeout signatures (tc_idx = None): the 16-byte digests are built on the GPU.
pub fn verify_tcs(tc_rounds: &[u64], pk: &[[u8; 32]], sig: &[[u8; 64]], high_qc_rounds: &[u64], tc_idx: Option<&[u32]>) -> Option<Vec<bool>> {
    let c = ctx()?;
    let mut tbm = vec![0u32; (tc_rounds.len() + 31) / 32 + 1];
    let rc = unsafe { hs_verify_tcs(c, tc_rounds.as_ptr(), tc_rounds.len(), pk.as_ptr() as *const u8, std::ptr::null(), sig.as_ptr() as *const u8,
                                    high_qc_rounds.as_ptr(), tc_idx.map_or(std::ptr::null(), |t| t.as_ptr()), sig.len(), std::ptr::null_mut(), tbm.as_mut_ptr()) };
    Some((0..tc_rounds.len()).map(|j| rc == HS_OK && tbm[j / 32] >> (j % 32) & 1 == 1).collect())
}
/// Digest = SHA-512[..32] of many messages (mempool/src/processor.rs:30 with several batches in flight).  None = hash on the CPU.
pub fn digest32_many(msgs: &[&[u8]]) -> Option<Vec<[u8; 32]>> {
    if msgs.len() < GPU_MIN_DIGEST_MSGS { return None; }
    let c = ctx()?;
    let mut off = Vec::with_capacity(msgs.len() + 1);
    let mut data = Vec::new();
    off.push(0u64);
    for m in msgs { data.extend_from_slice(m); off.push(data.len() as u64); }
    let mut out = vec![[0u8; 32]; msgs.len()];
    let rc = unsafe { hs_digest32_batch(c, data.as_ptr(), off.as_ptr(), msgs.len(), out.as_mut_ptr() as *mut u8) };
    if rc == HS_OK { Some(out) } else { None }   // a failed digest call falls back to the CPU hash: a digest has no "reject"
}

/// Everything `ingest_frames` extracted: frame i is group i of one hs_verify_groups pass.
pub struct Ingested { pub info: Vec<HsFrameInfo>, pub sig: Vec<u8>, pub pk: Vec<u8>, pub msg_idx: Vec<u32>, pub group_idx: Vec<u32>, pub mode: Vec<u8>,
                      pub preimages: Vec<u8>, pub pre_off: Vec<u64> }

/// Receiver side (consensus/src/consensus.rs:138): bincode `ConsensusMessage` frames -> flat arrays, without building the message
/// structs first.  Host-only (works without a GPU).  Malformed frames come back with kind == HS_FRAME_MALFORMED and no items.
pub fn ingest_frames(frames: &[&[u8]]) -> Result<Ingested, GpuError> {
    let n = frames.len();
    let mut off = Vec::with_capacity(n + 1);
    let mut blob = Vec::new();
    off.push(0u64);
    for f in frames { blob.extend_from_slice(f); off.push(blob.len() as u64); }
    let mut info = vec![HsFrameInfo::default(); n.max(1)];
    // every item costs >= 116 frame bytes and every preimage is copied from frame bytes: generous first guess, exact retry on NOMEM
    let (mut ci, mut cm, mut cp) = (blob.len() / 116 + n + 1, blob.len() / 60 + n + 1, blob.len() + 64 * n + 64);
    for _ in 0..2 {
        let mut g = Ingested { info: Vec::new(), sig: vec![0; ci * 64], pk: vec![0; ci * 32], msg_idx: vec![0; ci], group_idx: vec![0; ci], mode: vec![0; ci],
                               preimages: vec![0; cp], pre_off: vec![0; cm + 1] };
        let mut o = HsIngestOut { cap_items: ci, cap_msgs: cm, cap_pre_bytes: cp, sig: g.sig.as_mut_ptr(), pk: g.pk.as_mut_ptr(), msg_idx: g.msg_idx.as_mut_ptr(),
                                  group_idx: g.group_idx.as_mut_ptr(), mode: g.mode.as_mut_ptr(), preimages: g.preimages.as_mut_ptr(), pre_off: g.pre_off.as_mut_ptr(),
                                  n_items: 0, n_msgs: 0, pre_bytes: 0 };
        let rc = unsafe { hs_ingest_consensus_frames(blob.as_ptr(), off.as_ptr(), n, info.as_mut_ptr(), &mut o) };
        if rc == HS_OK {
            g.sig.truncate(o.n_items * 64); g.pk.truncate(o.n_items * 32); g.msg_idx.truncate(o.n_items); g.group_idx.truncate(o.n_items);
            g.mode.truncate(o.n_items); g.preimages.truncate(o.pre_bytes); g.pre_off.truncate(o.n_msgs + 1);
            info.truncate(n);
            g.info = info;
            return Ok(g);
        }
        if rc != HS_ERR_NOMEM { return Err(GpuError::Engine(format!("hs_ingest_consensus_frames: status {}", rc))); }
        ci = o.n_items + 1; cm = o.n_msgs + 1; cp = o.pre_bytes + 1;
    }
    Err(GpuError::Engine("ingest capacity retry failed".into()))
}
/// One GPU pass over everything `ingest_frames` found: bit j of the result = every signature of frame j verified (author strict, QC
/// votes by the batch equation, TC votes strict).  The stake / duplicate / genesis pre-checks of messages.rs stay with the caller, who
/// has the item ranges in `info`.  None = no GPU.
pub fn verify_ingested(g: &Ingested) -> Option<Vec<bool>> {
    let c = ctx()?;
    let n_groups = g.info.len();
    let mut gbm = vec![0u32; (n_groups + 31) / 32 + 1];
    let rc = unsafe { hs_verify_groups(c, g.preimages.as_ptr(), g.pre_off.as_ptr(), g.pre_off.len().saturating_sub(1), g.sig.as_ptr(), g.pk.as_ptr(), std::ptr::null(),
                                       g.msg_idx.as_ptr(), g.group_idx.as_ptr(), g.mode.as_ptr(), g.msg_idx.len(), n_groups, std::ptr::null_mut(), gbm.as_mut_ptr()) };
    Some((0..n_groups).map(|j| rc == HS_OK && g.info[j].kind != HS_FRAME_MALFORMED && gbm[j / 32] >> (j % 32) & 1 == 1).collect())
}
