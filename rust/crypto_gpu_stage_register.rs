// crypto/src/gpu/stage_register.rs — the staged registration (hs_committee_stage_register, include/hs_crypto.h), a submodule of
// crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  Its extern block is its own; tests/test_committee_stage_register_bindings.py checks it against
// the header.
//
// `stage_committee` works inside the slots and the window of the last registration.  An epoch change that needs more slots than the
// spares (HS_ERR_NOMEM), or a new per-key window, used to mean `register_committee` at the boundary: the device drained, every vote
// waiting for the whole build, and no committee at all if it failed.  This builds and proves the next committee's whole key store
// beside the live one during the last rounds of the epoch; `commit_registration` switches it in with one drain.
use std::os::raw::c_int;

use super::{commit_on, ctx, discard_on, last_error, scrub, GpuError, HsCtx, Staged, HS_OK, KEYS, STAGED};

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_committee_stage_register(ctx: *mut HsCtx, pks: *const u8, n: usize, key_bits: c_int, out_valid_bitmap: *mut u32,
                                   out_key_bits: *mut c_int) -> c_int;
}

/// hs_committee_stage_register on one context: the shim's own and, one per member, `multi::Multi`'s.  Returns the validity words and
/// the window the staged store was built at.
pub(super) fn stage_register_on(c: *mut HsCtx, keys: &[[u8; 32]], key_bits: i32) -> Result<(Vec<u32>, i32), GpuError> {
    let mut valid = vec![0u32; (keys.len() + 31) / 32];
    let mut bits: c_int = 0;
    let rc = unsafe { hs_committee_stage_register(c, keys.as_ptr() as *const u8, keys.len(), key_bits, valid.as_mut_ptr(), &mut bits) };
    if rc != HS_OK { return Err(GpuError::Engine(last_error(c))); }
    Ok((valid, bits))
}

/// Prepares the next epoch's committee as a whole new registration while this one verifies: every table is built and proved on the
/// GPU's lowest-priority stream, and nothing changes for verification until `commit_registration`.  `key_bits` 0 takes the widest
/// window that fits beside the live tables; 8..17 asks for that window.  Returns the window and the indices of keys that do not
/// decompress.  Blocks for the build (about 0.1 ms per key at 13-bit windows): call it from `spawn_blocking`.  On Err the live
/// committee is untouched; HS_ERR_NOMEM means the new tables do not fit beside it, so register at the boundary or ask for a narrower
/// window.
pub fn stage_register_committee(keys: &[[u8; 32]], key_bits: i32) -> Result<(i32, Vec<usize>), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut staged = STAGED.lock().unwrap();
    let (valid, bits) = stage_register_on(c, keys, key_bits)?;  // refused while a stage of either kind is pending
    *staged = Some(Staged::Registration(keys.to_vec()));
    Ok((bits, (0..keys.len()).filter(|i| valid[i / 32] >> (i % 32) & 1 == 0).collect()))
}

/// Switches the staged registration in at the epoch boundary (hs_committee_commit: one drain, no table built), then replaces the node's
/// map with the new keys and hands it to the scrub (hs_scrub_set_map).  A registration or update since the stage discarded it: Err,
/// and the map stays as it was.  A staged change is committed by `commit_committee` instead.  If the engine's commit fails, the stage
/// stays recorded: discard it.
pub fn commit_registration() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut keys = KEYS.lock().unwrap();  // held across the commit: the map and the engine change together
    let mut staged = STAGED.lock().unwrap();
    let staged_keys = match staged.as_ref() {
        Some(Staged::Registration(k)) => k.clone(),
        Some(Staged::Change { .. }) => return Err(GpuError::Engine("commit_registration: a committee change is staged (commit_committee)".into())),
        None => return Err(GpuError::Engine("commit_registration: nothing staged".into())),
    };
    commit_on(c)?;
    *staged = None;
    *keys = staged_keys.iter().map(|k| Some(*k)).collect();
    scrub::set_map(c, &keys)
}

/// Drops the staged registration (hs_committee_discard): its tables are freed.  A staged change is dropped by `discard_committee`.
pub fn discard_registration() -> Result<(), GpuError> {
    let c = ctx().ok_or(GpuError::Unavailable)?;
    let mut staged = STAGED.lock().unwrap();
    if let Some(Staged::Change { .. }) = *staged {
        return Err(GpuError::Engine("discard_registration: a committee change is staged (discard_committee)".into()));
    }
    discard_on(c)?;
    *staged = None;
    Ok(())
}
