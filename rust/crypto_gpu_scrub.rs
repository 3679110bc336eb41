// crypto/src/gpu/scrub.rs — the engine-owned scrub of the live key tables (hs_scrub_start, hs_scrub_set_map, hs_scrub_stats,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block passes a callback, so it is its own block; tests/test_scrub_bindings.py checks
// it against the header.
//
// `audit_tables` proves the tables at start-up and after each committee change.  Between those, a stray write by other CUDA code in
// the process could change a table entry, and that slot would give wrong verdicts until the next audit.  The scrub closes that window
// without a loop in the node: the engine's own thread audits a bounded slice of the tables per tick against the node's map, repairs
// what it finds, and calls back.  A repair that fails switches the GPU off, as a failed `audit_tables` does.
use std::os::raw::{c_int, c_void};
use std::sync::atomic::Ordering;

use super::{ctx, last_error, GpuError, HsCtx, DISABLED, HS_OK, KEYS};

/// hs_scrub_cb: runs on the scrub's thread once per tick that found anything (HS_AUDIT_* classes found, those its repair left).
pub type HsScrubCb = unsafe extern "C" fn(user: *mut c_void, found: u32, failed: u32, first_slot: usize);

/// A tick every 15.6 ms of 128 key slots and 2,883,585 base-point entries: a pass of a 4,096-key committee and the 24-bit base-point
/// table in 32 ticks, about half a second (DESIGN.md §5j has the measured cost of a tick and of a pass beside a vote burst).
pub const SCRUB_PERIOD_US: u32 = 15625;
pub const SCRUB_SLOTS_PER_TICK: u32 = 128;
pub const SCRUB_BASE_ENTRIES_PER_TICK: u32 = 2883585;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_scrub_start(ctx: *mut HsCtx, expect_pks: *const u8, expect_live: *const u32, n_slots: usize, period_us: u32, slots_per_tick: u32,
                      base_entries_per_tick: u32, cb_or_null: Option<HsScrubCb>, user: *mut c_void) -> c_int;
    fn hs_scrub_set_map(ctx: *mut HsCtx, expect_pks: *const u8, expect_live: *const u32, n_slots: usize) -> c_int;
    fn hs_scrub_stats(ctx: *mut HsCtx, out: *mut u64) -> c_int;
}

/// The node's index -> key map as the engine takes it: key bytes (zeros for a freed index) and the bitmap of live indices.
pub(crate) fn map_of(expected: &[Option<[u8; 32]>]) -> (Vec<u8>, Vec<u32>) {
    let pks: Vec<u8> = expected.iter().flat_map(|k| k.unwrap_or([0u8; 32])).collect();
    let mut live = vec![0u32; (expected.len() + 31) / 32];
    for (i, k) in expected.iter().enumerate() { if k.is_some() { live[i / 32] |= 1 << (i % 32); } }
    (pks, live)
}

unsafe extern "C" fn on_finding(_user: *mut c_void, _found: u32, failed: u32, _first_slot: usize) {
    // found alone: the engine repaired and re-proved what it found, and the caches of verified records were emptied; a corrected
    // signature-cache entry (HS_AUDIT_SIGCACHE) holds its re-checked flag byte and is never in failed
    if failed != 0 { DISABLED.store(true, Ordering::Release); }
}

/// Starts the scrub against the shim's map.  Call it once at start-up, after `register_committee` and `self_test`.  When the
/// node-wide queue's signature cache is on, each tick also re-checks a slice of it (`sig_audit::attach`).
pub fn start() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let keys = KEYS.lock().unwrap();
    let (pks, live) = map_of(&keys);
    let rc = unsafe { hs_scrub_start(c, if keys.is_empty() { std::ptr::null() } else { pks.as_ptr() }, live.as_ptr(), keys.len(), SCRUB_PERIOD_US,
                                     SCRUB_SLOTS_PER_TICK, SCRUB_BASE_ENTRIES_PER_TICK, Some(on_finding), std::ptr::null_mut()) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    super::sig_audit::attach();
    Ok(())
}

/// Gives the scrub the map after a committee change (the shim calls it with KEYS held); until then the scrub pauses.
pub(crate) fn set_map(c: *mut HsCtx, expected: &[Option<[u8; 32]>]) -> Result<(), GpuError> {
    let (pks, live) = map_of(expected);
    let rc = unsafe { hs_scrub_set_map(c, if expected.is_empty() { std::ptr::null() } else { pks.as_ptr() }, live.as_ptr(), expected.len()) };
    if rc == HS_OK { Ok(()) } else { Err(GpuError::Engine(last_error(c))) }
}

/// The scrub's counters for the node's metrics: passes, slots audited, base entries audited, ticks, findings, slots repaired, failed
/// repairs, ticks paused.  None when there is no GPU.
pub fn stats() -> Option<[u64; 8]> {
    let c = ctx()?;
    let mut out = [0u64; 8];
    if unsafe { hs_scrub_stats(c, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
