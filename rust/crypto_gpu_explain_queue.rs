// crypto/src/gpu/explain_queue.rs — the explain lane of the node-wide verify queue (hs_queue_explain, hs_queue_submit_explain,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block passes a callback and a user pointer, so it is its own block;
// tests/test_explain_queue_bindings.py checks it against the header.
//
// explain_rejected_queued: why a rejected message was rejected, awaited instead of blocking.  The synchronous `explain_rejected` holds
// the context's mutex for its whole re-check (about 1.4 ms), and every vote launch of the queue needs that mutex to enqueue, so a peer
// sending junk could stall the votes.  Through the lane the mutex is held only to enqueue, the re-check runs on a bounded share of the
// SMs at the lowest priority, and one launch explains every pending request, so every rejected record of the message is explained at
// once for about the cost of one.
use std::os::raw::{c_int, c_void};
use std::sync::atomic::{AtomicBool, Ordering};
use std::sync::Once;
use tokio::sync::oneshot;

use super::queue::{queue, HsQueue, HsQueueCb};
use super::{Explained, HsRec128, HS_MODE_BATCH_EQ, HS_OK, HS_WHY_A_SMALL, HS_WHY_R_SMALL};

/// Limits of one explain request on the node-wide queue: every record of a 10,000-validator Block with its TC (about 13,300
/// signatures, 1.7 MB of region), with room to spare.
pub const EXPLAIN_MAX_RECORDS: usize = 16_384;
pub const EXPLAIN_MAX_BYTES: usize = 4 << 20;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_explain(q: *mut HsQueue, max_records: usize, max_bytes: usize) -> c_int;
    fn hs_queue_submit_explain(q: *mut HsQueue, recs: *const HsRec128, n: usize, cb_or_null: Option<HsQueueCb>, user: *mut c_void,
                               out_ticket: *mut usize) -> c_int;
}

static ENABLE: Once = Once::new();
static ENABLED: AtomicBool = AtomicBool::new(false);

/// Turns the explain lane on for the node-wide queue, once.  False when it could not be (no pinned or device memory): callers then
/// keep the rejection unexplained.
pub(crate) fn enable(q: *mut HsQueue, max_records: usize, max_bytes: usize) -> bool {
    ENABLE.call_once(|| ENABLED.store(unsafe { hs_queue_explain(q, max_records, max_bytes) } == HS_OK, Ordering::Release));
    ENABLED.load(Ordering::Acquire)
}

struct Pending { tx: oneshot::Sender<Option<Vec<u8>>>, n: usize }

unsafe extern "C" fn on_done(user: *mut c_void, _ticket: usize, status: c_int, bitmap: *const u32) {
    let p = Box::from_raw(user as *mut Pending);
    // an engine failure explains nothing: None, and the rejection stands
    let out = if status == HS_OK {
        Some((0..p.n).map(|i| (*bitmap.add(i / 4) >> (8 * (i % 4))) as u8).collect())
    } else {
        None
    };
    let _ = p.tx.send(out);  // the awaiting task may have been dropped: nothing to do
}

/// Explains a rejected message through the queue: `recs` are its records, `modes` their verdict modes (HS_MODE_*) and `verdicts` the
/// bits the engine returned for them.  Every rejected record goes into ONE explain request; the result holds one `Explained` per
/// rejected record, in record order, with `engine_fault` set exactly as `explain_rejected` sets it (the re-check finds the record valid
/// in its own mode: audit and repair the tables, and answer the message on the dalek path).  None = no record was rejected, no GPU, no
/// lane, inconsistent arrays, more than the lane's limits, no arena room right now (back-pressure), or an engine failure: keep the
/// rejection unexplained.  An explanation is advisory; None never changes a verdict.
pub async fn explain_rejected_queued(recs: &[HsRec128], modes: &[u8], verdicts: &[bool]) -> Option<Vec<Explained>> {
    if modes.len() != recs.len() || verdicts.len() != recs.len() { return None; }
    let index: Vec<usize> = (0..recs.len()).filter(|&i| !verdicts[i]).collect();
    if index.is_empty() || index.len() > EXPLAIN_MAX_RECORDS { return None; }
    let rejected: Vec<HsRec128> = index.iter().map(|&i| recs[i]).collect();
    let rx = {
        let q = queue()?;
        if !enable(q, EXPLAIN_MAX_RECORDS, EXPLAIN_MAX_BYTES) { return None; }
        let (tx, rx) = oneshot::channel();
        let user = Box::into_raw(Box::new(Pending { tx, n: rejected.len() })) as *mut c_void;
        let rc = unsafe { hs_queue_submit_explain(q, rejected.as_ptr(), rejected.len(), Some(on_done), user, std::ptr::null_mut()) };
        if rc != HS_OK {
            drop(unsafe { Box::from_raw(user as *mut Pending) });  // not queued: the callback never runs
            return None;                                          // HS_ERR_NOMEM is back-pressure, HS_ERR_ARG a bad request
        }
        rx
    };  // (no raw pointer lives across the await: the future stays Send)
    let why = rx.await.ok().flatten()?;
    Some(index.iter().zip(why).map(|(&i, why)| {
        let valid = if modes[i] == HS_MODE_BATCH_EQ { why & !(HS_WHY_A_SMALL | HS_WHY_R_SMALL) == 0 } else { why == 0 };
        Explained { index: i, why, engine_fault: valid }
    }).collect())
}
