// crypto/src/gpu/groups_dev.rs — the device-resident certificate pass (hs_verify_groups_dev, include/hs_crypto.h), a submodule of
// crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block takes device pointers and a stream (`void *` in C), so it is its own block;
// tests/test_groups_dev.py checks it against the header.
//
// For a node that keeps its certificate arrays in HBM (its own CUDA allocator, or one rank of a multi-GPU process group): a Block's
// author signature, QC votes and TC votes, or a view-change burst of Timeouts with their high_qcs, verified without a host round trip.
// The calls only enqueue; item verdicts (each in its own mode) are in `item_bitmap` once `stream` has run the pass, and group verdicts
// come from the per-group AND over them (hs_qc_and_dev, `group_and_dev`).
use std::os::raw::{c_int, c_void};

use super::{HsCtx, HS_OK};

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_verify_groups_dev(ctx: *mut HsCtx, preimages: *const c_void, pre_off: *const c_void, n_msgs: usize, sig: *const c_void,
                            pk_or_null: *const c_void, validator_idx_or_null: *const c_void, msg_idx: *const c_void, mode_or_null: *const c_void,
                            n_items: usize, item_bitmap: *mut c_void, stream: *mut c_void) -> c_int;
    fn hs_qc_and_dev(ctx: *mut HsCtx, vote_bitmap: *const c_void, qc_idx: *const c_void, n_votes: usize, n_qc: usize, qc_bitmap: *mut c_void,
                     stream: *mut c_void) -> c_int;
}

/// Device arrays of one pass, laid out as hs_verify_groups_dev reads them.  `pk` null = committee-indexed (`validator_idx`);
/// `mode` null = every item strict.
pub struct DevGroups {
    pub preimages: *const c_void, pub pre_off: *const c_void, pub n_msgs: usize, pub sig: *const c_void, pub pk: *const c_void,
    pub validator_idx: *const c_void, pub msg_idx: *const c_void, pub mode: *const c_void, pub n_items: usize,
}

/// Enqueues the pass on `stream`.  Err = nothing was enqueued for it: reject every item.
///
/// # Safety
/// Every pointer is device memory of the context's GPU holding what `DevGroups` describes (the engine does not check device
/// arrays), and sig / keys / modes stay valid until the stream has run the pass.
pub unsafe fn verify_groups_dev(ctx: *mut HsCtx, g: &DevGroups, item_bitmap: *mut c_void, stream: *mut c_void) -> Result<(), super::GpuError> {
    let rc = hs_verify_groups_dev(ctx, g.preimages, g.pre_off, g.n_msgs, g.sig, g.pk, g.validator_idx, g.msg_idx, g.mode, g.n_items, item_bitmap, stream);
    if rc == HS_OK { Ok(()) } else { Err(super::GpuError::Engine(super::last_error(ctx))) }
}

/// Enqueues the group verdicts on `stream`: bit j of `group_bitmap` = AND of the item bits whose `group_idx` (u32 per item) is j, 1 for a
/// group with no items.  Pass the item bitmap of `verify_groups_dev` (or the gathered one of every rank).  Err = reject every group.
///
/// # Safety
/// Device pointers of the context's GPU: `item_bitmap` with n_items bits, `group_idx` with n_items entries < n_groups, `group_bitmap`
/// with (n_groups + 31) / 32 words.
pub unsafe fn group_and_dev(ctx: *mut HsCtx, item_bitmap: *const c_void, group_idx: *const c_void, n_items: usize, n_groups: usize,
                            group_bitmap: *mut c_void, stream: *mut c_void) -> Result<(), super::GpuError> {
    let rc = hs_qc_and_dev(ctx, item_bitmap, group_idx, n_items, n_groups, group_bitmap, stream);
    if rc == HS_OK { Ok(()) } else { Err(super::GpuError::Engine(super::last_error(ctx))) }
}
