// crypto/src/gpu/msgs_queue.rs — whole certificates through the verify queue of libhs_crypto.so with their signed preimages
// instead of their Digests (hs_queue_submit_msgs, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block passes a callback and a user pointer, so it is its own block;
// tests/test_msgs_queue_bindings.py checks it against the header.
//
// verify_msgs_queued: every signature of ONE consensus message as one request, called from the connection tasks.  The caller
// passes the preimages each signature is over (a TC vote's 16-byte round || high_qc_round, a QC's 40-byte hash || round, the
// Block::digest preimage) and the GPU computes the Digests, so the task hashes nothing on its own thread: a TC of N - f votes
// costs N - f SHA-512 calls less before the request enters the ring.  The arrays are exactly what `ingest_frames` in the shim
// writes for one frame (the receiver path: ingest one frame -> verify_msgs_queued).
//
// verify_timeout_queued: Timeout::verify as one request, the author's signature plus its high_qc's votes.  The node-wide queue
// keeps a certificate cache (cert_cache.rs), so the QC that every Timeout of a view change carries is verified once and each
// further Timeout costs one ring record, its author's.
use std::os::raw::{c_int, c_void};
use tokio::sync::oneshot;

use super::cert_cache;
use super::group_queue::GROUP_MAX_SIGS;
use super::queue::{queue, HsQueue, HsQueueCb};
use super::HS_OK;

/// The node-wide queue with its certificate cache on, so that the Blocks' QCs warm it for the Timeouts that carry them.
fn cached_queue() -> Option<*mut HsQueue> {
    let q = queue()?;
    cert_cache::enable(q);
    Some(q)
}

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_queue_submit_msgs(q: *mut HsQueue, preimages: *const u8, pre_off: *const u64, n_msgs: usize, sig: *const u8, pk: *const u8,
                            msg_idx: *const u32, modes_or_null: *const u8, n: usize, cb_or_null: Option<HsQueueCb>, user: *mut c_void,
                            out_ticket: *mut usize) -> c_int;
}

struct Pending { tx: oneshot::Sender<Vec<bool>>, n: usize }

unsafe extern "C" fn on_done(user: *mut c_void, _ticket: usize, status: c_int, bitmap: *const u32) {
    let p = Box::from_raw(user as *mut Pending);
    // an engine failure rejects every signature of the certificate (core.rs drops a message on any Err)
    let bits = (0..p.n).map(|i| status == HS_OK && *bitmap.add(i / 32) >> (i % 32) & 1 == 1).collect();
    let _ = p.tx.send(bits);  // the awaiting task may have been dropped: nothing to do
}

/// One message's signatures (1..=GROUP_MAX_SIGS records, the cut-over of `group_queue`) through the queue: record i is
/// (sig[64 i ..], pk[32 i ..]) over Digest(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]]), judged by modes[i] = 0
/// (Signature::verify) or 1 (the verify_batch condition).  None = use the synchronous path (no GPU, an oversized or inconsistent
/// request, or no room in the ring or the preimage arena right now); Some(bits) = per-record verdicts.
pub async fn verify_msgs_queued(preimages: &[u8], pre_off: &[u64], sig: &[u8], pk: &[u8], msg_idx: &[u32], modes: &[u8]) -> Option<Vec<bool>> {
    let n = msg_idx.len();
    if n == 0 || n > GROUP_MAX_SIGS || modes.len() != n || sig.len() != 64 * n || pk.len() != 32 * n || pre_off.len() < 2 { return None; }
    if pre_off.last().map_or(true, |&end| end as usize > preimages.len()) { return None; }
    submit(preimages, pre_off, sig, pk, msg_idx, modes).await
}

/// Timeout::verify (messages.rs:250-265) through the queue: record 0 is the author's signature (strict) over `author_pre`
/// (round || high_qc.round, 16 bytes), records 1.. are the high_qc's votes (the verify_batch condition) over `qc_pre`
/// (hash || round, 40 bytes); a genesis high_qc has no votes.  Not bound by GROUP_MAX_SIGS: with the cache on, a QC that is
/// already verified or in flight takes no ring records, so a Timeout normally costs one.  None = use the synchronous path (no GPU,
/// inconsistent arrays, or no room in the ring or the preimage arena right now); Some(bits) = record 0 then the votes.
pub async fn verify_timeout_queued(author_pre: &[u8], author_sig: &[u8; 64], author_pk: &[u8; 32], qc_pre: &[u8],
                                   votes: &[([u8; 32], [u8; 64])]) -> Option<Vec<bool>> {
    let n = 1 + votes.len();
    let mut preimages = Vec::with_capacity(author_pre.len() + qc_pre.len());
    preimages.extend_from_slice(author_pre);
    preimages.extend_from_slice(qc_pre);
    let pre_off = [0, author_pre.len() as u64, preimages.len() as u64];
    let (mut sig, mut pk) = (Vec::with_capacity(64 * n), Vec::with_capacity(32 * n));
    sig.extend_from_slice(author_sig);
    pk.extend_from_slice(author_pk);
    for (v_pk, v_sig) in votes {
        pk.extend_from_slice(v_pk);
        sig.extend_from_slice(v_sig);
    }
    let msg_idx: Vec<u32> = (0..n).map(|i| (i > 0) as u32).collect();
    let modes: Vec<u8> = (0..n).map(|i| (i > 0) as u8).collect();
    submit(&preimages, &pre_off, &sig, &pk, &msg_idx, &modes).await
}

async fn submit(preimages: &[u8], pre_off: &[u64], sig: &[u8], pk: &[u8], msg_idx: &[u32], modes: &[u8]) -> Option<Vec<bool>> {
    let n = msg_idx.len();
    let rx = {
        let q = cached_queue()?;
        let (tx, rx) = oneshot::channel();
        let user = Box::into_raw(Box::new(Pending { tx, n })) as *mut c_void;
        let rc = unsafe {
            hs_queue_submit_msgs(q, preimages.as_ptr(), pre_off.as_ptr(), pre_off.len() - 1, sig.as_ptr(), pk.as_ptr(), msg_idx.as_ptr(),
                                 modes.as_ptr(), n, Some(on_done), user, std::ptr::null_mut())
        };
        if rc != HS_OK {
            drop(unsafe { Box::from_raw(user as *mut Pending) });  // not queued: the callback never runs
            return None;                                          // HS_ERR_NOMEM is back-pressure, HS_ERR_ARG a bad frame
        }
        rx
    };  // (no raw pointer lives across the await: the future stays Send)
    rx.await.ok()
}
