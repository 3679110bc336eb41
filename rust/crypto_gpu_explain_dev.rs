// crypto/src/gpu/explain_dev.rs — the explanation of a device-resident pass's rejected items (hs_explain_groups_dev,
// include/hs_crypto.h), a submodule of crypto_gpu_shim.rs beside `groups_dev`, whose `DevGroups` it takes.
//
// STATUS: source only, like the shim.  Its extern block is its own; tests/test_explain_dev.py checks it against the header.
//
// `explain_rejected` tells a false reject from a bad signature for a message verified through host memory.  A pass whose arrays stay in
// HBM (`groups_dev::verify_groups_dev`, one rank of a sharded pass) gets the same answer here, with nothing copied back but the four
// out words the node chooses to read.
use std::os::raw::{c_int, c_void};

use super::groups_dev::DevGroups;
use super::{GpuError, HsCtx, HS_OK};

/// hs_explain_groups_dev's why byte of an item it did not examine (accepted, or past the cap).
pub const HS_WHY_NOT_EXAMINED: u8 = 0x80;
/// Words of hs_explain_groups_dev's out array.
pub const HS_EXPLAIN_DEV_OUT: usize = 4;

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_explain_groups_dev(ctx: *mut HsCtx, preimages: *const c_void, pre_off: *const c_void, n_msgs: usize, sig: *const c_void,
                             pk: *const c_void, msg_idx: *const c_void, mode_or_null: *const c_void, item_bitmap: *const c_void,
                             n_items: usize, max_explain: usize, why: *mut c_void, out: *mut c_void, stream: *mut c_void) -> c_int;
}

/// Enqueues on `stream` the table-free re-check of the lowest-index `max_explain` items (0 = all) whose bit in `item_bitmap` is 0, for
/// the pass `g` describes.  Once the stream has run it, `why` (n_items bytes) holds each examined item's HS_WHY_* mask and
/// HS_WHY_NOT_EXAMINED elsewhere, and `out` (HS_EXPLAIN_DEV_OUT u32 words) holds: [0] items whose bit is 0, [1] items examined,
/// [2] engine faults (items the pass rejected that the re-check finds valid in their mode), [3] the lowest faulting index
/// (u32::MAX: none).
///
/// A non-zero out[2] means the engine, not the signer, is wrong.  The node then audits and repairs its tables (`audit_tables`),
/// re-checks the signature cache (`sig_audit::audit_cache`), and answers the messages holding those items on the dalek path instead
/// of dropping them.  A zero out[2] confirms every examined rejection: log the masks with the messages and drop them.
///
/// `g.pk` must hold key bytes.  For a committee-indexed pass, gather the node's own index -> key map by validator index into a device
/// array and pass that, so the check does not read the tables it doubts.  Err = nothing was enqueued: keep the rejections.
///
/// # Safety
/// Every pointer is device memory of the context's GPU: `g` as for `verify_groups_dev`, `item_bitmap` with g.n_items bits, `why` with
/// g.n_items bytes and `out` with HS_EXPLAIN_DEV_OUT words, all valid until the stream has run the call.
pub unsafe fn explain_rejected_dev(ctx: *mut HsCtx, g: &DevGroups, item_bitmap: *const c_void, max_explain: usize, why: *mut c_void,
                                   out: *mut c_void, stream: *mut c_void) -> Result<(), GpuError> {
    let rc = hs_explain_groups_dev(ctx, g.preimages, g.pre_off, g.n_msgs, g.sig, g.pk, g.msg_idx, g.mode, item_bitmap, g.n_items, max_explain,
                                   why, out, stream);
    if rc == HS_OK { Ok(()) } else { Err(GpuError::Engine(super::last_error(ctx))) }
}
