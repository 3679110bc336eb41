// crypto/src/gpu/mend.rs — the mend of corrupt comb-table entries in place (hs_table_mend, hs_table_mend_stats, hs_scrub_mend,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block is its own; tests/test_table_mend_bindings.py checks it against the header.
//
// A repair rebuilds a corrupt base-point table with the device drained (about 0.2 s with no vote verified) and takes a validator whose
// table is corrupt out of service until its whole table is rebuilt and proved.  The mend recomputes only the windows the audit flags,
// off the table, and stores only the entries that differ: verification goes on and every slot stays in service.  It cannot fix key
// bytes, flag bytes or the hash table; what it leaves goes to `audit_tables`, which repairs.
use std::os::raw::c_int;

use super::{ctx, last_error, GpuError, HsCtx, HS_ERR_SELFTEST, HS_OK, KEYS};

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_table_mend(ctx: *mut HsCtx, expect_pks: *const u8, expect_live: *const u32, n_slots: usize, out_slot_bits: *mut u8,
                     out_found: *mut u32, out_left: *mut u32) -> c_int;
    fn hs_table_mend_stats(ctx: *mut HsCtx, out: *mut u64) -> c_int;
    fn hs_scrub_mend(ctx: *mut HsCtx, on: c_int) -> c_int;
}

/// Mends the tables against the node's map; returns the HS_AUDIT_* classes it found.  What it leaves (key bytes, flag bytes, lookup
/// entries, or an entry the mend could not fix) goes on to `audit_tables`, the repair, which switches the GPU off if that fails too.
pub fn mend_tables(expected: &[Option<[u8; 32]>]) -> Result<u32, GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let (pks, live) = super::scrub::map_of(expected);
    let (mut found, mut left) = (0u32, 0u32);
    let rc = unsafe { hs_table_mend(c, if expected.is_empty() { std::ptr::null() } else { pks.as_ptr() }, live.as_ptr(), expected.len(),
                                    std::ptr::null_mut(), &mut found, &mut left) };
    if rc == HS_OK { return Ok(found); }
    if rc == HS_ERR_SELFTEST { return super::audit_tables(expected).map(|_| found); }
    Err(GpuError::Engine(last_error(c)))
}

/// Lets the scrub mend what it can instead of repairing it: `scrub::start` keeps the repair as the default, and the node calls this
/// once after it.  A tick with a finding the mend cannot fix still repairs.
pub fn attach_scrub() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let _keys = KEYS.lock().unwrap();  // the same order as the scrub's start and map changes
    if unsafe { hs_scrub_mend(c, 1) } == HS_OK { Ok(()) } else { Err(GpuError::Engine(last_error(c))) }
}

/// The mend's counters for the node's metrics: calls, windows recomputed, entries rewritten, windows left, slots left to repair,
/// cache flushes.  None when there is no GPU.
pub fn stats() -> Option<[u64; 6]> {
    let c = ctx()?;
    let mut out = [0u64; 6];
    if unsafe { hs_table_mend_stats(c, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
