// crypto/src/gpu/sig_share.rs — sharing of the node-wide verify queue's signature cache with the synchronous verify calls and the
// queue's batch lane (hs_queue_sig_share, hs_queue_sig_share_stats, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes the queue's handle, so it is its own block;
// tests/test_sig_share_bindings.py checks it against the header.
//
// TCs and Blocks above GROUP_MAX_SIGS go to hs_verify_tcs / hs_verify_groups under spawn_blocking, and a collected burst of Timeouts
// goes to the batch lane.  With sharing on, both answer the votes the queue already verified from the queue's table, and the strict
// records they verify go into it, so the TC after a burst and the Block that carries the TC are probes.  Verdicts do not change.
use std::os::raw::c_int;

use super::queue::HsQueue;
use super::HS_OK;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_sig_share(q: *mut HsQueue, on: c_int) -> c_int;
    fn hs_queue_sig_share_stats(q: *mut HsQueue, out: *mut u64) -> c_int;
}

/// Shares the node-wide queue's signature cache; called once, right after the cache is turned on.  A failure leaves sharing off:
/// the synchronous calls and the lane then verify every record, with the same verdicts.
pub(crate) fn enable(q: *mut HsQueue) {
    let _ = unsafe { hs_queue_sig_share(q, 1) };
}

/// The shared passes' counters for the node's metrics: records probed, hits, inserts, inserts that evicted a live entry, shared
/// passes.  None when there is no GPU queue.
pub fn sig_share_stats() -> Option<[u64; 5]> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 5];
    if unsafe { hs_queue_sig_share_stats(q, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
