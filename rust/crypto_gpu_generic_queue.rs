// crypto/src/gpu/generic_queue.rs — the generic-key device path of the node-wide verify queue (hs_queue_generic,
// hs_queue_generic_stats, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes the queue's handle, so it is its own block;
// tests/test_generic_queue_bindings.py checks it against the header.
//
// The queue's device path needs every key of a request in the registered committee.  Any other request (the node has not
// registered yet, its table budget was too small to register, or a validator joined `Committee` before hs_committee_update ran)
// used to be verified synchronously on the queue's thread, and every vote queued behind it waited that long.  With the option on,
// such requests are verified by a queue kernel on the GPU, on the queue's lower-priority stream, and the votes' launches go on.
// Verdicts are those of the queue without it.
use std::os::raw::c_int;
use std::sync::Once;

use super::queue::HsQueue;
use super::HS_OK;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_generic(q: *mut HsQueue, on: c_int) -> c_int;
    fn hs_queue_generic_stats(q: *mut HsQueue, out: *mut u64) -> c_int;
}

static ENABLE: Once = Once::new();

/// Turns the generic path on for the node-wide queue, once.  A failure leaves it off: those requests then take the synchronous
/// path on the queue's thread, with the same verdicts.
pub(crate) fn enable(q: *mut HsQueue) {
    ENABLE.call_once(|| { let _ = unsafe { hs_queue_generic(q, 1) }; });
}

/// The generic path's counters for the node's metrics: launches, records they carried, requests.  None when there is no GPU
/// queue.
pub fn generic_stats() -> Option<[u64; 3]> {
    let q = super::queue::queue()?;
    let mut out = [0u64; 3];
    if unsafe { hs_queue_generic_stats(q, out.as_mut_ptr()) } == HS_OK { Some(out) } else { None }
}
