// crypto/src/gpu/group_queue.rs — whole certificates through the verify queue of libhs_crypto.so (hs_queue_submit_group,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block passes a callback and a user pointer, so it is its own block;
// tests/test_group_queue_bindings.py checks it against the header.
//
// verify_group_queued: every signature of ONE consensus message as one request, called from the connection tasks
// (consensus.rs ConsensusReceiverHandler::dispatch) — a Block (author strict + QC votes batch-eq + TC votes strict,
// messages.rs:54-76), a Timeout with its high_qc (:250-265), a TC (:290-315).  It goes into the node-wide queue of
// `queue::verify_queued`, so a replica's Block::verify shares launches with the vote burst instead of holding the engine's
// mutex for a synchronous call, and the awaiting task does not block its runtime worker thread.
use std::os::raw::{c_int, c_void};
use tokio::sync::oneshot;

use super::queue::{queue, HsQueue, HsQueueCb};
use super::{HsRec128, HS_OK};

/// Largest certificate sent through the queue: the largest measured size at which one queued request was no slower than the
/// synchronous calls (strict author verify + verify_batch) — tools/replay_config5.cpp "replica_block", one H100 80GB HBM3 at a
/// 400 W power limit, p50 over 20 blocks: 502 records (N = 750) 243 us queued vs 286 us synchronous; 668 records (N = 1,000)
/// 304 us vs 297 us; 1,002 records (N = 1,500, the queue's bulk kernel) 327 us vs 316 us; 6,668 records (N = 10,000) 728 us
/// vs 469 us.  Larger certificates use the synchronous batch front ends.  At 4 records (N = 4) the two took 141 us and 142 us;
/// they stay on the queue, which does not block a runtime worker while they verify.
pub const GROUP_MAX_SIGS: usize = 502;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_submit_group(q: *mut HsQueue, recs: *const HsRec128, n: usize, modes_or_null: *const u8, cb_or_null: Option<HsQueueCb>,
                             user: *mut c_void, out_ticket: *mut usize) -> c_int;
}

struct Pending { tx: oneshot::Sender<Vec<bool>>, n: usize }

unsafe extern "C" fn on_done(user: *mut c_void, _ticket: usize, status: c_int, bitmap: *const u32) {
    let p = Box::from_raw(user as *mut Pending);
    // an engine failure rejects every signature of the certificate (core.rs drops a message on any Err)
    let bits = (0..p.n).map(|i| status == HS_OK && *bitmap.add(i / 32) >> (i % 32) & 1 == 1).collect();
    let _ = p.tx.send(bits);  // the awaiting task may have been dropped: nothing to do
}

/// One message's signatures (1..=GROUP_MAX_SIGS records) through the queue; modes[i] = 0 (Signature::verify) or 1 (the
/// verify_batch condition) for record i.  None = use the synchronous path (no GPU, an oversized request, mismatched modes, or no
/// room in the ring right now); Some(bits) = per-record verdicts, identical to verify_strict_many / the batch condition per record.
pub async fn verify_group_queued(recs: &[HsRec128], modes: &[u8]) -> Option<Vec<bool>> {
    if recs.is_empty() || recs.len() > GROUP_MAX_SIGS || modes.len() != recs.len() { return None; }
    let rx = {
        let q = queue()?;
        let (tx, rx) = oneshot::channel();
        let user = Box::into_raw(Box::new(Pending { tx, n: recs.len() })) as *mut c_void;
        let rc = unsafe {
            hs_queue_submit_group(q, recs.as_ptr(), recs.len(), modes.as_ptr(), Some(on_done), user, std::ptr::null_mut())
        };
        if rc != HS_OK {
            drop(unsafe { Box::from_raw(user as *mut Pending) });  // not queued: the callback never runs
            return None;                                          // HS_ERR_NOMEM is back-pressure: verify synchronously
        }
        rx
    };  // (no raw pointer lives across the await: the future stays Send)
    rx.await.ok()
}
