// crypto/src/gpu/sig_audit.rs — the audit of the node-wide verify queue's signature cache (hs_queue_sig_audit, hs_queue_sig_audit_stats,
// hs_scrub_sig_cache, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes the queue's handle, so it is its own block;
// tests/test_sig_audit_bindings.py checks it against the header.
//
// With the cache and its sharing on, every TC vote and most Block votes are answered from the stored flag byte of a cache entry, with
// no check at all.  A flipped bit there is a false accept (a batch-eq-only record answered strict) or a false reject that the table
// audit cannot see, since no table is wrong.  The audit re-checks each held entry from its 128 bytes, table-free, and corrects the flag
// bytes that disagree.  The scrub runs it a slice per tick; `engine_fault` runs it over the whole table beside `audit_tables`.
use std::os::raw::c_int;

use super::queue::HsQueue;
use super::{ctx, HsCtx, HS_OK};

/// Buckets of the cache each scrub tick re-checks: 512 of the 16,384 (2,048 entries) is a pass of the node's table in 32 ticks, about
/// half a second at the scrub's 15.6 ms period, the pace of the table scrub (DESIGN.md §5k has the cost of a slice beside a vote burst).
pub const SIG_AUDIT_BUCKETS_PER_TICK: u32 = 512;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_sig_audit(q: *mut HsQueue, first_bucket: usize, n_buckets: usize, out: *mut u64) -> c_int;
    fn hs_queue_sig_audit_stats(q: *mut HsQueue, out: *mut u64) -> c_int;
    fn hs_scrub_sig_cache(ctx: *mut HsCtx, q_or_null: *mut HsQueue, buckets_per_tick: u32) -> c_int;
}

/// Attaches the node-wide queue's cache to the context's scrub when the cache is on: `scrub::start` calls it, and so does
/// `sig_cache::enable` when the cache comes on later (the attachment outlives a scrub restart).  A failure leaves the cache to
/// `audit_cache` alone.
pub(crate) fn attach() {
    if !super::sig_cache::is_on() { return; }
    if let (Some(c), Some(q)) = (ctx(), super::queue::queue()) {
        let _ = unsafe { hs_scrub_sig_cache(c, q, SIG_AUDIT_BUCKETS_PER_TICK) };
    }
}

/// Re-checks the whole cache and corrects what it finds (the `engine_fault` branch calls it beside `audit_tables`): a false reject
/// answered from a flipped flag byte then clears.  Returns the entries corrected; None when there is no GPU queue or its cache is off.
pub fn audit_cache() -> Option<u64> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 7];
    if unsafe { hs_queue_sig_audit(q, 0, 0, out.as_mut_ptr()) } == HS_OK { Some(out[1]) } else { None }
}

/// The audit's counters for the node's metrics: audits, entries re-checked, corrected, skipped, full passes.  None when there is no GPU
/// queue.
pub fn stats() -> Option<[u64; 5]> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 5];
    if unsafe { hs_queue_sig_audit_stats(q, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
