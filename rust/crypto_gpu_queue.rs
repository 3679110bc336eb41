// crypto/src/gpu/queue.rs — the verify queue of libhs_crypto.so (hs_queue_*, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  The queue's FFI passes a callback and a user pointer, so it has its own extern block;
// tests/test_queue_bindings.py checks that block against the header (the shim's block is checked by test_binding_consistency.py).
//
// verify_queued: the lone Signature::verify of Vote::verify (one per incoming vote at the leader), Timeout::verify and the Block
// author check, called from many tasks at once (one per peer connection, consensus.rs ConsensusReceiverHandler::dispatch).  Every
// call goes into ONE node-wide queue; its dispatcher thread gathers whatever is pending into a single latency-path launch, so
// concurrent connections share launches instead of queueing behind each other.  Each caller awaits only its own verdicts.
use std::os::raw::{c_int, c_void};
use std::sync::OnceLock;
use tokio::sync::oneshot;

use super::{ctx, HsCtx, HsRec128, HS_OK};

#[repr(C)] pub struct HsQueue { _private: [u8; 0] }
/// hs_queue_cb: runs once per request on the queue's thread.
pub type HsQueueCb = unsafe extern "C" fn(user: *mut c_void, ticket: usize, status: c_int, bitmap: *const u32);
/// Largest request the queue takes (one message's signatures); larger sets use the batch front ends of the shim.
pub const QUEUE_MAX_SIGS: usize = 64;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_create(ctx: *mut HsCtx, ring_records: usize, out: *mut *mut HsQueue) -> c_int;
    fn hs_queue_submit(q: *mut HsQueue, recs: *const HsRec128, n: usize, mode: u32, cb_or_null: Option<HsQueueCb>, user: *mut c_void,
                       out_ticket: *mut usize) -> c_int;
}

struct Queue(*mut HsQueue);
unsafe impl Send for Queue {}
unsafe impl Sync for Queue {}          // hs_queue_submit is thread-safe and never blocks
static QUEUE: OnceLock<Option<Queue>> = OnceLock::new();

/// The node-wide queue on the shim's context (default ring of 4,096 records); lives as long as the process.  Shared with the
/// certificate requests of `group_queue::verify_group_queued`.
pub(crate) fn queue() -> Option<*mut HsQueue> {
    QUEUE.get_or_init(|| {
        let c = ctx()?;
        let mut q = std::ptr::null_mut();
        if unsafe { hs_queue_create(c, 0, &mut q) } != HS_OK || q.is_null() { return None; }
        super::generic_queue::enable(q);
        Some(Queue(q))
    }).as_ref().map(|q| q.0)
}

struct Pending { tx: oneshot::Sender<Vec<bool>>, n: usize }

unsafe extern "C" fn on_done(user: *mut c_void, _ticket: usize, status: c_int, bitmap: *const u32) {
    let p = Box::from_raw(user as *mut Pending);
    // an engine failure rejects every signature of the request (core.rs drops a message on any Err)
    let bits = (0..p.n).map(|i| status == HS_OK && *bitmap.add(i / 32) >> (i % 32) & 1 == 1).collect();
    let _ = p.tx.send(bits);  // the awaiting task may have been dropped: nothing to do
}

/// Signature::verify (mode 0) or the verify_batch condition (mode 1) of one message's 1..=64 signatures through the queue.
/// None = use the CPU path (no GPU, an oversized request, or the ring is full right now); Some(bits) = verdicts, identical to
/// verify_strict_many on the same records.
pub async fn verify_queued(recs: &[HsRec128], mode: u32) -> Option<Vec<bool>> {
    if recs.is_empty() || recs.len() > QUEUE_MAX_SIGS { return None; }
    let rx = {
        let q = queue()?;
        let (tx, rx) = oneshot::channel();
        let user = Box::into_raw(Box::new(Pending { tx, n: recs.len() })) as *mut c_void;
        let rc = unsafe { hs_queue_submit(q, recs.as_ptr(), recs.len(), mode, Some(on_done), user, std::ptr::null_mut()) };
        if rc != HS_OK {
            drop(unsafe { Box::from_raw(user as *mut Pending) });  // not queued: the callback never runs
            return None;                                          // HS_ERR_NOMEM is back-pressure: verify this one on the CPU
        }
        rx
    };  // (no raw pointer lives across the await: the future stays Send)
    rx.await.ok()
}
