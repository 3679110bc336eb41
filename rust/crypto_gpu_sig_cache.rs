// crypto/src/gpu/sig_cache.rs — the signature cache of the node-wide verify queue (hs_queue_sig_cache, hs_queue_sig_stats,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes the queue's handle, so it is its own block;
// tests/test_sig_cache_bindings.py checks it against the header.
//
// A TC's votes are the author signatures of the Timeouts that preceded it, and the Block after it carries the same TC.  With the
// cache on, the queue's kernels keep every record they accepted (signature, key bytes and Digest), so those votes are probes that
// hit instead of verifies.  Verdicts are those of the queue without it.
use std::os::raw::c_int;
use std::sync::atomic::{AtomicBool, Ordering};
use std::sync::Once;

use super::queue::HsQueue;
use super::HS_OK;

/// Records the node-wide queue's table holds (16,384 buckets of 4 entries, 592 bytes a bucket: 9.7 MB).  A view change of N validators inserts about N Timeout
/// author records, so this keeps several view changes at N = 10,000.
pub const SIG_CACHE_ENTRIES: usize = 1 << 16;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_sig_cache(q: *mut HsQueue, entries: usize) -> c_int;
    fn hs_queue_sig_stats(q: *mut HsQueue, out: *mut u64) -> c_int;
}

static ENABLE: Once = Once::new();
static ON: AtomicBool = AtomicBool::new(false);

/// Turns the cache on for the node-wide queue, once, and then shares it with the synchronous calls and the batch lane
/// (`sig_share::enable`) and attaches it to the scrub (`sig_audit::attach`).  A failure leaves it off: every record is then verified,
/// with the same verdicts.
pub(crate) fn enable(q: *mut HsQueue) {
    ENABLE.call_once(|| {
        if unsafe { hs_queue_sig_cache(q, SIG_CACHE_ENTRIES) } == HS_OK {
            super::sig_share::enable(q);
            ON.store(true, Ordering::Release);
            super::sig_audit::attach();
        }
    });
}

/// Whether `enable` turned the cache on.
pub(crate) fn is_on() -> bool { ON.load(Ordering::Acquire) }

/// The cache's counters for the node's metrics: records probed, hits, inserts, inserts that evicted a live entry, entries held.
/// None when there is no GPU queue.
pub fn sig_stats() -> Option<[u64; 5]> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 5];
    if unsafe { hs_queue_sig_stats(q, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
