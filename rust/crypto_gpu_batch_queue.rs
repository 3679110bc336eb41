// crypto/src/gpu/batch_queue.rs — the batch lane of the node-wide verify queue (hs_queue_batch, hs_queue_submit_batch,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block passes a callback and a user pointer, so it is its own block;
// tests/test_batch_queue_bindings.py checks it against the header.
//
// verify_groups_queued: a whole hs_verify_groups pass (a Block of a large committee with its QC and TC, or a view-change burst
// collected in `Core`, one group per certificate) as ONE queue request that a task awaits.  It runs the throughput kernels of the
// synchronous call on the lane's own stream and scratch, and the context's mutex is held only while its launches are enqueued, so
// the votes' launches go on meanwhile.  No thread blocks on it: it replaces `tokio::task::spawn_blocking` around the synchronous call.
use std::os::raw::{c_int, c_void};
use std::sync::atomic::{AtomicBool, Ordering};
use std::sync::Once;
use tokio::sync::oneshot;

use super::queue::{queue, HsQueue, HsQueueCb};
use super::HS_OK;

/// Limits of one batch request on the node-wide queue: a 10,000-validator Block carrying a TC (about 13,300 signatures and
/// 1.6 MB of region), or a 10,000-validator view-change burst, with room to spare.
pub const BATCH_MAX_ITEMS: usize = 32_768;
pub const BATCH_MAX_BYTES: usize = 8 << 20;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_batch(q: *mut HsQueue, max_items: usize, max_bytes: usize) -> c_int;
    fn hs_queue_submit_batch(q: *mut HsQueue, preimages: *const u8, pre_off: *const u64, n_msgs: usize, sig: *const u8, pk: *const u8,
                             msg_idx: *const u32, group_idx: *const u32, modes_or_null: *const u8, n_items: usize, n_groups: usize,
                             cb_or_null: Option<HsQueueCb>, user: *mut c_void, out_ticket: *mut usize) -> c_int;
}

static ENABLE: Once = Once::new();
static ENABLED: AtomicBool = AtomicBool::new(false);

/// Turns the batch lane on for the node-wide queue, once.  False when it could not be (no pinned or device memory): callers then
/// keep the synchronous path.
pub(crate) fn enable(q: *mut HsQueue, max_items: usize, max_bytes: usize) -> bool {
    ENABLE.call_once(|| ENABLED.store(unsafe { hs_queue_batch(q, max_items, max_bytes) } == HS_OK, Ordering::Release));
    ENABLED.load(Ordering::Acquire)
}

struct Pending { tx: oneshot::Sender<Option<(Vec<bool>, Vec<bool>)>>, n_items: usize, n_groups: usize }

unsafe extern "C" fn on_done(user: *mut c_void, _ticket: usize, status: c_int, bitmap: *const u32) {
    let p = Box::from_raw(user as *mut Pending);
    // an engine failure is None: the caller rejects every certificate of the batch (core.rs drops a message on any Err)
    let out = if status == HS_OK {
        let bit = |w: usize, i: usize| *bitmap.add(w + i / 32) >> (i % 32) & 1 == 1;
        let gw = (p.n_groups + 31) / 32;
        Some(((0..p.n_groups).map(|j| bit(0, j)).collect(), (0..p.n_items).map(|i| bit(gw, i)).collect()))
    } else {
        None
    };
    let _ = p.tx.send(out);  // the awaiting task may have been dropped: nothing to do
}

/// hs_verify_groups with key bytes, awaited instead of blocking: item i is (sig[64 i ..], pk[32 i ..]) over
/// Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]]) in group group_idx[i], judged by modes[i] = 0
/// (Signature::verify) or 1 (the verify_batch condition).  Some((group bits, item bits)) = the verdicts, bit for bit those of the
/// synchronous call.  None = not verified here (no GPU, no lane, inconsistent arrays, more than the lane's limits, no arena room right
/// now, or an engine failure): verify synchronously.  None is never an accept.
pub async fn verify_groups_queued(preimages: &[u8], pre_off: &[u64], sig: &[u8], pk: &[u8], msg_idx: &[u32], group_idx: &[u32], modes: &[u8],
                                  n_groups: usize) -> Option<(Vec<bool>, Vec<bool>)> {
    let n = msg_idx.len();
    if n == 0 || n_groups == 0 || n > BATCH_MAX_ITEMS || group_idx.len() != n || modes.len() != n || sig.len() != 64 * n || pk.len() != 32 * n
        || pre_off.len() < 2 { return None; }
    if pre_off.last().map_or(true, |&end| end as usize > preimages.len()) { return None; }
    let rx = {
        let q = queue()?;
        if !enable(q, BATCH_MAX_ITEMS, BATCH_MAX_BYTES) { return None; }
        let (tx, rx) = oneshot::channel();
        let user = Box::into_raw(Box::new(Pending { tx, n_items: n, n_groups })) as *mut c_void;
        let rc = unsafe {
            hs_queue_submit_batch(q, preimages.as_ptr(), pre_off.as_ptr(), pre_off.len() - 1, sig.as_ptr(), pk.as_ptr(), msg_idx.as_ptr(),
                                  group_idx.as_ptr(), modes.as_ptr(), n, n_groups, Some(on_done), user, std::ptr::null_mut())
        };
        if rc != HS_OK {
            drop(unsafe { Box::from_raw(user as *mut Pending) });  // not queued: the callback never runs
            return None;                                          // HS_ERR_NOMEM is back-pressure, HS_ERR_ARG a bad batch
        }
        rx
    };  // (no raw pointer lives across the await: the future stays Send)
    rx.await.ok().flatten()
}
