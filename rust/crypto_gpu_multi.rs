// crypto/src/gpu/multi.rs — several GPUs from the node's one process (hs_multi_*, include/hs_crypto.h), a submodule of crypto_gpu_shim.rs.
//
// STATUS: source only, like the shim.  `hs_multi` is a handle type of its own, so this module has its own extern block;
// tests/test_multi_bindings.py checks it against the header.
//
// The node's Core task and its mempool Processors call `crypto` from one process.  A `Multi` over the node's GPUs shards every large
// host-pointer verify (hs_multi_verify_*: contiguous 32-aligned record ranges, one per member) and runs smaller calls whole on one member,
// chosen round-robin, so the tasks' small calls land on different GPUs.  Verdicts equal the single-context calls bit for bit.
use std::os::raw::{c_char, c_int};

use super::{GpuError, HsCtx, HsRec128, HS_OK};

#[repr(C)] pub struct HsMulti { _private: [u8; 0] }

#[link(name = "hs_crypto")]
extern "C" {
    fn hs_multi_create(out: *mut *mut HsMulti, devices: *const c_int, n_devices: usize, flags: u32) -> c_int;
    fn hs_multi_destroy(m: *mut HsMulti);
    fn hs_multi_last_error(m: *const HsMulti) -> *const c_char;
    fn hs_multi_members(m: *const HsMulti) -> usize;
    fn hs_multi_member(m: *mut HsMulti, i: usize) -> *mut HsCtx;
    fn hs_multi_committee_register(m: *mut HsMulti, pks: *const u8, n: usize, out_valid_bitmap: *mut u32) -> c_int;
    fn hs_multi_committee_update(m: *mut HsMulti, add_pks: *const u8, n_add: usize, remove_idx: *const u32, n_remove: usize,
                                 out_add_idx: *mut u32) -> c_int;
    fn hs_multi_verify_rec128(m: *mut HsMulti, recs: *const HsRec128, n: usize, mode: u32, out_bitmap: *mut u32) -> c_int;
    fn hs_multi_verify_msgs(m: *mut HsMulti, sig: *const u8, pk: *const u8, vidx: *const u32, msgs: *const u8, msg_len: usize, n: usize, mode: u32,
                            out_bitmap: *mut u32) -> c_int;
    fn hs_multi_verify_groups(m: *mut HsMulti, preimages: *const u8, pre_off: *const u64, n_msgs: usize, sig: *const u8, pk: *const u8,
                              vidx: *const u32, msg_idx: *const u32, group_idx: *const u32, mode: *const u8, n_items: usize, n_groups: usize,
                              out_item_bitmap: *mut u32, out_group_bitmap: *mut u32) -> c_int;
}

/// Owner of one hs_multi.  Calls from several threads are safe: sharded calls serialise on the multi-context, small ones on a member.
pub struct Multi(*mut HsMulti);
unsafe impl Send for Multi {}
unsafe impl Sync for Multi {}

impl Drop for Multi {
    fn drop(&mut self) { unsafe { hs_multi_destroy(self.0) } }   // joins the workers, destroys the members and their queues
}

/// A member context handed to a staging thread (each call is serialised on the member's own mutex).
struct Member(*mut HsCtx);
unsafe impl Send for Member {}
unsafe impl Sync for Member {}

fn bits(bm: &[u32], n: usize) -> Vec<bool> { (0..n).map(|i| bm[i / 32] >> (i % 32) & 1 == 1).collect() }

impl Multi {
    /// One member per entry of `devices` (a device may repeat); `flags` as hs_ctx_create.
    pub fn new(devices: &[i32], flags: u32) -> Result<Multi, GpuError> {
        let mut p = std::ptr::null_mut();
        let rc = unsafe { hs_multi_create(&mut p, devices.as_ptr(), devices.len(), flags) };
        if rc == HS_OK && !p.is_null() { Ok(Multi(p)) } else { Err(GpuError::Unavailable) }
    }
    fn err(&self) -> GpuError {
        GpuError::Engine(unsafe { std::ffi::CStr::from_ptr(hs_multi_last_error(self.0)).to_string_lossy().into_owned() })
    }
    pub fn members(&self) -> usize { unsafe { hs_multi_members(self.0) } }
    /// Member i for the single-device calls (a verify queue, say).  Borrowed: never register a committee on it directly.
    pub fn member(&self, i: usize) -> *mut HsCtx { unsafe { hs_multi_member(self.0, i) } }

    /// The same committee on every member.  Keys that do not decompress are reported as in `register_committee`.
    pub fn register_committee(&self, keys: &[[u8; 32]]) -> Result<(), GpuError> {
        let mut valid = vec![0u32; (keys.len() + 31) / 32];
        let rc = unsafe { hs_multi_committee_register(self.0, keys.as_ptr() as *const u8, keys.len(), valid.as_mut_ptr()) };
        if rc != HS_OK { return Err(self.err()); }
        let bad: Vec<usize> = (0..keys.len()).filter(|i| valid[i / 32] >> (i % 32) & 1 == 0).collect();
        if bad.is_empty() { Ok(()) } else { Err(GpuError::InvalidKeys(bad)) }
    }
    /// Incremental epoch change on every member: the added validators' indices, the same on each.  Err: re-register.
    pub fn update_committee(&self, add: &[[u8; 32]], remove_idx: &[u32]) -> Result<Vec<u32>, GpuError> {
        let mut out = vec![0u32; add.len().max(1)];
        let rc = unsafe { hs_multi_committee_update(self.0, add.as_ptr() as *const u8, add.len(), remove_idx.as_ptr(), remove_idx.len(), out.as_mut_ptr()) };
        if rc != HS_OK { return Err(self.err()); }
        out.truncate(add.len());
        Ok(out)
    }
    /// The staged committee change on every member, member by member through the single-context calls (as a repair is): stages on
    /// every member at once, one thread each, and returns the added validators' indices.  If any member fails, or the members return
    /// different indices, the stage is discarded on every member and Err returned: nothing stays staged.
    pub fn stage_committee(&self, add: &[[u8; 32]], remove_idx: &[u32]) -> Result<Vec<u32>, GpuError> {
        let members: Vec<Member> = (0..self.members()).map(|i| Member(self.member(i))).collect();
        let res: Vec<Result<Vec<u32>, GpuError>> = std::thread::scope(|s| {
            let hs: Vec<_> = members.iter().map(|m| s.spawn(move || { let m: &Member = m; super::stage_on(m.0, add, remove_idx) })).collect();
            hs.into_iter().map(|h| h.join().unwrap_or(Err(GpuError::Unavailable))).collect()
        });
        let (mut idx, mut fail): (Option<Vec<u32>>, Option<GpuError>) = (None, None);
        for r in res {
            match r {
                Err(e) => { if fail.is_none() { fail = Some(e); } }
                Ok(v) => match &idx {
                    None => idx = Some(v),
                    Some(x) if *x == v => {}
                    Some(_) => { if fail.is_none() { fail = Some(GpuError::Engine("stage_committee: the members gave different indices".into())); } }
                },
            }
        }
        match fail {
            None => Ok(idx.unwrap_or_default()),
            Some(e) => {
                for m in &members { let _ = super::discard_on(m.0); }
                Err(e)
            }
        }
    }
    /// The staged registration on every member, member by member through the single-context call: stages on every member at once,
    /// one thread each, and returns the window and the indices of keys that do not decompress.  If any member fails, or the members
    /// differ in validity or window, the stage is discarded on every member and Err returned: every member keeps its committee.
    /// `commit_committee` switches it in.
    pub fn stage_register_committee(&self, keys: &[[u8; 32]], key_bits: i32) -> Result<(i32, Vec<usize>), GpuError> {
        let members: Vec<Member> = (0..self.members()).map(|i| Member(self.member(i))).collect();
        let res: Vec<Result<(Vec<u32>, i32), GpuError>> = std::thread::scope(|s| {
            let hs: Vec<_> = members.iter()
                .map(|m| s.spawn(move || { let m: &Member = m; super::stage_register::stage_register_on(m.0, keys, key_bits) })).collect();
            hs.into_iter().map(|h| h.join().unwrap_or(Err(GpuError::Unavailable))).collect()
        });
        let (mut got, mut fail): (Option<(Vec<u32>, i32)>, Option<GpuError>) = (None, None);
        for r in res {
            match r {
                Err(e) => { if fail.is_none() { fail = Some(e); } }
                Ok(v) => match &got {
                    None => got = Some(v),
                    Some(x) if *x == v => {}
                    Some(_) => { if fail.is_none() { fail = Some(GpuError::Engine("stage_register_committee: the members gave different validity or windows".into())); } }
                },
            }
        }
        match (fail, got) {
            (None, Some((valid, bits))) => Ok((bits, (0..keys.len()).filter(|i| valid[i / 32] >> (i % 32) & 1 == 0).collect())),
            (fail, _) => {
                for m in &members { let _ = super::discard_on(m.0); }
                Err(fail.unwrap_or(GpuError::Unavailable))
            }
        }
    }
    /// Commits the staged change on every member.  Err: the members may differ, re-register.
    pub fn commit_committee(&self) -> Result<(), GpuError> {
        (0..self.members()).try_for_each(|i| super::commit_on(self.member(i)))
    }
    /// Discards the staged change on every member.
    pub fn discard_committee(&self) -> Result<(), GpuError> {
        (0..self.members()).try_for_each(|i| super::discard_on(self.member(i)))
    }
    /// hs_verify_rec128 across the members.  An engine failure rejects everything.
    pub fn verify_rec128(&self, recs: &[HsRec128], mode: u32) -> Vec<bool> {
        let mut bm = vec![0u32; (recs.len() + 31) / 32];
        let rc = unsafe { hs_multi_verify_rec128(self.0, recs.as_ptr(), recs.len(), mode, bm.as_mut_ptr()) };
        if rc == HS_OK { bits(&bm, recs.len()) } else { vec![false; recs.len()] }
    }
    /// hs_verify_msgs across the members: n messages of msg_len bytes, key bytes (`pk`, 32 per message) or committee indices.
    pub fn verify_msgs(&self, sig: &[u8], pk: Option<&[u8]>, vidx: Option<&[u32]>, msgs: &[u8], msg_len: usize, mode: u32) -> Vec<bool> {
        let n = sig.len() / 64;
        if msg_len == 0 || msgs.len() != n * msg_len || pk.map_or(false, |k| k.len() != 32 * n) || vidx.map_or(false, |v| v.len() != n) || (pk.is_none() && vidx.is_none()) {
            return vec![false; n];
        }
        let mut bm = vec![0u32; (n + 31) / 32];
        let rc = unsafe { hs_multi_verify_msgs(self.0, sig.as_ptr(), pk.map_or(std::ptr::null(), |k| k.as_ptr()), vidx.map_or(std::ptr::null(), |v| v.as_ptr()),
                                               msgs.as_ptr(), msg_len, n, mode, bm.as_mut_ptr()) };
        if rc == HS_OK { bits(&bm, n) } else { vec![false; n] }
    }
    /// `verify_ingested` across the members: bit j = every signature of frame j verified.
    pub fn verify_ingested(&self, g: &super::Ingested) -> Vec<bool> {
        let n_groups = g.info.len();
        let mut gbm = vec![0u32; (n_groups + 31) / 32 + 1];
        let rc = unsafe { hs_multi_verify_groups(self.0, g.preimages.as_ptr(), g.pre_off.as_ptr(), g.pre_off.len().saturating_sub(1), g.sig.as_ptr(), g.pk.as_ptr(),
                                                 std::ptr::null(), g.msg_idx.as_ptr(), g.group_idx.as_ptr(), g.mode.as_ptr(), g.msg_idx.len(), n_groups,
                                                 std::ptr::null_mut(), gbm.as_mut_ptr()) };
        (0..n_groups).map(|j| rc == HS_OK && g.info[j].kind != super::HS_FRAME_MALFORMED && gbm[j / 32] >> (j % 32) & 1 == 1).collect()
    }
}
