// crypto/src/gpu/cert_cache.rs — the certificate cache of the node-wide verify queue (hs_queue_cert_cache, hs_queue_cert_stats,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes the queue's handle, so it is its own block;
// tests/test_cert_cache_bindings.py checks it against the header.
//
// During a view change every validator's Timeout carries the same high_qc.  With the cache on, the queue verifies that QC's
// votes once: a Timeout whose QC is in flight in an earlier request waits for it, and one whose QC already verified (the Block
// that carried it, or an earlier Timeout) is answered from the cache.  Either way it puts one record in the ring, its author's.
use std::os::raw::c_int;
use std::sync::Once;

use super::queue::HsQueue;
use super::HS_OK;

/// Bytes of verified certificates the node-wide queue keeps: a QC of 2f + 1 votes takes 9 + 40 + 96 (2f + 1) bytes, so about
/// 25 QCs at N = 10,000 and 250 at N = 1,000.
pub const CERT_CACHE_BYTES: usize = 16 << 20;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_cert_cache(q: *mut HsQueue, max_bytes: usize) -> c_int;
    fn hs_queue_cert_stats(q: *mut HsQueue, out: *mut u64) -> c_int;
}

static ENABLE: Once = Once::new();

/// Turns the cache on for the node-wide queue, once, and the queue's signature cache with it.  A failure leaves a cache off:
/// every request is then verified in full, with the same verdicts.
pub(crate) fn enable(q: *mut HsQueue) {
    ENABLE.call_once(|| { let _ = unsafe { hs_queue_cert_cache(q, CERT_CACHE_BYTES) }; });
    super::sig_cache::enable(q);
}

/// The cache's counters for the node's metrics: spans looked up, hits, in-flight joins, records answered without verifying them,
/// spans inserted, bytes held.  None when there is no GPU queue.
pub fn cert_stats() -> Option<[u64; 6]> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 6];
    if unsafe { hs_queue_cert_stats(q, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
