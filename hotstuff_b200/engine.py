"""Engine: Python handle on one hs_ctx (one CUDA device).  Thin: marshals numpy / torch buffers into the C ABI.

Host-side mirror of the reference interface lives in crypto.py; this module is the batch surface the consensus call
sites would use (QC/TC vote sets, mempool batch digests) plus device-resident entry points for the benchmark.
"""
import ctypes
import threading

import numpy as np

from . import _lib

MODE_STRICT = 0    # Signature::verify      (crypto/src/lib.rs:200-204)
MODE_BATCH_EQ = 1  # Signature::verify_batch (crypto/src/lib.rs:206-219), per-signature condition
HS_ERR_SELFTEST = 4  # hs_self_test: a path gave a wrong answer
# hs_explain_rec128: one bit per check of the decision procedure a record fails (include/hs_crypto.h)
WHY_S_NONCANONICAL = 1  # S >= l
WHY_A_INVALID = 2       # A does not decompress
WHY_R_INVALID = 4       # R does not decompress
WHY_A_SMALL = 8         # [8]A is the identity
WHY_R_SMALL = 16        # [8]R is the identity
WHY_EQUATION = 32       # S, A, R parse and [S]B + [k](-A) != R
WHY_NOT_EXAMINED = 0x80  # hs_explain_groups_dev only: the item was accepted, or is past max_explain
EXPLAIN_DEV_OUT = 4      # hs_explain_groups_dev's out words
AUDIT_SIGCACHE = 32  # a scrub callback's found: the tick corrected a signature-cache entry (hs_scrub_sig_cache)


class EngineError(RuntimeError):
    pass


def _ptr(a):
    if a is None:
        return None
    return a.ctypes.data_as(ctypes.c_void_p)


def _u8(a, shape_last=None):
    a = np.ascontiguousarray(np.frombuffer(a, dtype=np.uint8) if isinstance(a, (bytes, bytearray, memoryview)) else a, dtype=np.uint8)
    if shape_last is not None and a.size % shape_last:
        raise ValueError("buffer length is not a multiple of %d" % shape_last)
    return a


def bitmap_to_bools(bitmap, n):
    return np.unpackbits(bitmap.view(np.uint8), bitorder="little")[:n].astype(bool)


class Engine:
    def __init__(self, device=0, base_window=0, key_window=0, key_cache=True):
        """base_window / key_window: comb window widths in bits (0 = engine defaults: 24 and the widest that fits).
        key_cache: learn tables for unregistered keys between calls (include/hs_crypto.h, hs_cached_keys)."""
        self.lib = _lib.load()
        h = ctypes.c_void_p()
        rc = self.lib.hs_ctx_create(ctypes.byref(h), int(device), (int(base_window) & 0xff) | ((int(key_window) & 0xff) << 8) | (0 if key_cache else 0x10000))
        if rc != 0 or not h:
            raise EngineError("hs_ctx_create(device=%d) failed with status %d (no GPU / CUDA error); there is no CPU fallback" % (device, rc))
        self.h = h
        self.device = int(device)
        self.n_keys = 0
        self._queues = []
        self._owned = True

    @classmethod
    def _view(cls, lib, h, device):
        """A non-owning Engine on a context another object owns (MultiEngine.member): close() leaves the context alone."""
        e = cls.__new__(cls)
        e.lib, e.h, e.device, e.n_keys, e._queues, e._owned = lib, h, int(device), 0, [], False
        return e

    def close(self):
        for q in list(getattr(self, "_queues", [])):
            q.close()
        if getattr(self, "h", None):
            if getattr(self, "_owned", True):
                self.lib.hs_ctx_destroy(self.h)
            self.h = None

    def queue(self, ring_records=0):
        """A VerifyQueue on this context (hs_queue_create): concurrent small verifies share latency-path launches."""
        return VerifyQueue(self, ring_records)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed: status %d: %s" % (what, rc, self.lib.hs_last_error(self.h).decode()))

    @property
    def cached_keys(self):
        return int(self.lib.hs_cached_keys(self.h))

    @property
    def window_bits(self):
        """(per-key comb window bits or 0, base-point comb window bits)"""
        a, b = ctypes.c_int(0), ctypes.c_int(0)
        self.lib.hs_window_bits(self.h, ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value

    @property
    def kernel_launches(self):
        return int(self.lib.hs_kernel_launches(self.h))

    def self_test(self, key_bits=0, recs=None, expect=None):
        """Known-answer self-test of every device path at this context's geometry (hs_self_test).  recs: (n,128) uint8 records and
        expect: n bytes (bit 0 strict, bit 1 batch-eq), or None for the built-in set; key_bits: 0 = the per-key window in use, 8..17 to
        force one.  Returns the mask of failing paths (HS_SELFTEST_* bits; 0 = every answer right, hs_last_error names the first
        mismatch otherwise).  Raises EngineError on a bad argument, no device memory for the scratch tables or a CUDA error."""
        failed = ctypes.c_uint32(0)
        if recs is None:
            rc = self.lib.hs_self_test(self.h, int(key_bits), None, None if expect is None else _ptr(_u8(expect)), 0, ctypes.byref(failed))
        else:
            recs = _u8(recs, 128).reshape(-1, 128)
            exp = None if expect is None else _u8(expect)
            rc = self.lib.hs_self_test(self.h, int(key_bits), _ptr(recs), _ptr(exp), recs.shape[0], ctypes.byref(failed))
        if rc == HS_ERR_SELFTEST:
            return int(failed.value)
        self._check(rc, "hs_self_test")
        return 0

    @property
    def key_slots(self):
        """Key slots in use (hs_key_slots): the committee's, spares taken by updates included, or the key cache's learned keys."""
        return int(self.lib.hs_key_slots(self.h))

    def table_audit(self, expect=None, live=None):
        """Audit of the live key tables on the GPU (hs_table_audit).  expect: (key_slots, 32) uint8, the node's index -> key map, or None
        to check the engine against itself; live: a uint32 bitmap of the slots expected live (None: every slot).  Returns (failed,
        slot_bits): the HS_AUDIT_* mask (0 = every check passed, last_error names the first finding otherwise) and one uint8 of
        HS_AUDIT_* bits per slot.  Raises EngineError on a bad argument (key_slots changed, expect given for key-cache tables), when the
        tables changed while the audit ran (call again), and on no memory or a CUDA error."""
        n = self.key_slots if expect is None else _u8(expect, 32).reshape(-1, 32).shape[0]
        exp = None if expect is None else _u8(expect, 32).reshape(-1, 32)
        lv = None if live is None else np.ascontiguousarray(live, dtype=np.uint32)
        if lv is not None and lv.size < (n + 31) // 32:
            raise ValueError("table_audit: %d live words for %d slots" % (lv.size, n))
        bits = np.zeros(max(1, n), dtype=np.uint8)
        failed = ctypes.c_uint32(0)
        rc = self.lib.hs_table_audit(self.h, _ptr(exp) if n and exp is not None else None, _ptr(lv) if lv is not None and lv.size else None, n,
                                     _ptr(bits), ctypes.byref(failed))
        if rc != HS_ERR_SELFTEST:
            self._check(rc, "hs_table_audit")
        return int(failed.value), bits[:n]

    def table_repair(self, expect=None, live=None):
        """Repair of what the audit finds (hs_table_repair), from the same authority: expect / live as for table_audit, else the engine's
        host mirror.  Returns (found, failed, slot_bits): the HS_AUDIT_* classes the first audit found, those the final audit still finds
        (0 = every finding repaired; last_error names the first one left otherwise) and the first audit's uint8 of HS_AUDIT_* bits per
        slot, i.e. the slots repaired.  Raises EngineError as table_audit does."""
        n = self.key_slots if expect is None else _u8(expect, 32).reshape(-1, 32).shape[0]
        exp = None if expect is None else _u8(expect, 32).reshape(-1, 32)
        lv = None if live is None else np.ascontiguousarray(live, dtype=np.uint32)
        if lv is not None and lv.size < (n + 31) // 32:
            raise ValueError("table_repair: %d live words for %d slots" % (lv.size, n))
        bits = np.zeros(max(1, n), dtype=np.uint8)
        found, failed = ctypes.c_uint32(0), ctypes.c_uint32(0)
        rc = self.lib.hs_table_repair(self.h, _ptr(exp) if n and exp is not None else None, _ptr(lv) if lv is not None and lv.size else None, n,
                                      _ptr(bits), ctypes.byref(found), ctypes.byref(failed))
        if rc != HS_ERR_SELFTEST:
            self._check(rc, "hs_table_repair")
        return int(found.value), int(failed.value), bits[:n]

    def table_mend(self, expect=None, live=None):
        """Mend of corrupt comb-table entries in place (hs_table_mend): recomputes the windows the audit flags off the table and stores
        only the entries that differ, with no drain and no slot out of service.  expect / live as for table_audit.  Returns (found, left,
        slot_bits): the HS_AUDIT_* classes the audit found, those left for table_repair (0 = everything mended; KEY, FLAG and LOOKUP
        findings are always left) and the audit's uint8 of HS_AUDIT_* bits per slot.  Raises EngineError as table_audit does."""
        n = self.key_slots if expect is None else _u8(expect, 32).reshape(-1, 32).shape[0]
        exp = None if expect is None else _u8(expect, 32).reshape(-1, 32)
        lv = None if live is None else np.ascontiguousarray(live, dtype=np.uint32)
        if lv is not None and lv.size < (n + 31) // 32:
            raise ValueError("table_mend: %d live words for %d slots" % (lv.size, n))
        bits = np.zeros(max(1, n), dtype=np.uint8)
        found, left = ctypes.c_uint32(0), ctypes.c_uint32(0)
        rc = self.lib.hs_table_mend(self.h, _ptr(exp) if n and exp is not None else None, _ptr(lv) if lv is not None and lv.size else None, n,
                                    _ptr(bits), ctypes.byref(found), ctypes.byref(left))
        if rc != HS_ERR_SELFTEST:
            self._check(rc, "hs_table_mend")
        return int(found.value), int(left.value), bits[:n]

    MEND_STATS = ("calls", "windows_recomputed", "entries_rewritten", "windows_left", "slots_left", "cache_flushes")

    def mend_stats(self):
        """The mend's counters (hs_table_mend_stats), the scrub's mends included, as a dict keyed by MEND_STATS."""
        out = (ctypes.c_uint64 * len(self.MEND_STATS))()
        self._check(self.lib.hs_table_mend_stats(self.h, out), "hs_table_mend_stats")
        return dict(zip(self.MEND_STATS, (int(v) for v in out)))

    def scrub_mend(self, on=True):
        """With on, a scrub tick whose findings can all be mended mends them (table_mend) instead of repairing them (hs_scrub_mend)."""
        self._check(self.lib.hs_scrub_mend(self.h, 1 if on else 0), "hs_scrub_mend")

    SCRUB_STATS = ("passes", "slots_audited", "base_entries_audited", "ticks", "findings", "slots_repaired", "failed_repairs",
                   "ticks_paused")

    def _scrub_map(self, expect, live, what):
        n = self.key_slots if expect is None else _u8(expect, 32).reshape(-1, 32).shape[0]
        exp = None if expect is None else _u8(expect, 32).reshape(-1, 32)
        lv = None if live is None else np.ascontiguousarray(live, dtype=np.uint32)
        if lv is not None and lv.size < (n + 31) // 32:
            raise ValueError("%s: %d live words for %d slots" % (what, lv.size, n))
        return n, exp, lv, (_ptr(exp) if n and exp is not None else None), (_ptr(lv) if lv is not None and lv.size else None)

    def scrub_start(self, expect=None, live=None, period_us=15625, slots_per_tick=128, base_entries_per_tick=2883585, callback=None):
        """Starts the engine-owned scrub of the live key tables (hs_scrub_start): every period_us a thread audits the next slots_per_tick
        key slots in service and base_entries_per_tick entries of the base-point table against expect / live (as for table_audit; None:
        the engine's host mirror), repairs what it finds and calls callback(found, failed, first_slot) once per tick that found anything,
        on the scrub's thread.  After a committee change it pauses until scrub_set_map.  The defaults make a pass of a 4,096-key
        committee and the 24-bit base-point table 32 ticks, about half a second (DESIGN.md §5j).  Raises EngineError when a scrub
        already runs or the map breaks the audit's rules."""
        n, exp, lv, p_exp, p_lv = self._scrub_map(expect, live, "scrub_start")
        cb = None
        if callback is not None:
            cb = _lib.SCRUB_CB(lambda user, found, failed, first_slot: callback(int(found), int(failed), int(first_slot)))
        rc = self.lib.hs_scrub_start(self.h, p_exp, p_lv, n, int(period_us), int(slots_per_tick), int(base_entries_per_tick),
                                     ctypes.cast(cb, ctypes.c_void_p) if cb is not None else None, None)
        self._check(rc, "hs_scrub_start")
        self._scrub_keep = (cb, exp, lv)  # the trampoline lives as long as the thread that calls it

    def scrub_set_map(self, expect=None, live=None):
        """The map of the slots after a committee change (hs_scrub_set_map): the paused scrub resumes with a new pass."""
        n, exp, lv, p_exp, p_lv = self._scrub_map(expect, live, "scrub_set_map")
        self._check(self.lib.hs_scrub_set_map(self.h, p_exp, p_lv, n), "hs_scrub_set_map")

    def scrub_stop(self):
        """Stops the scrub and joins its thread (hs_scrub_stop); a no-op when none runs."""
        self._check(self.lib.hs_scrub_stop(self.h), "hs_scrub_stop")

    def scrub_stats(self):
        """The scrub's counters (hs_scrub_stats) as a dict keyed by SCRUB_STATS."""
        out = (ctypes.c_uint64 * len(self.SCRUB_STATS))()
        self._check(self.lib.hs_scrub_stats(self.h, out), "hs_scrub_stats")
        return dict(zip(self.SCRUB_STATS, (int(v) for v in out)))

    def scrub_sig_cache(self, queue, buckets_per_tick=512):
        """Attaches a VerifyQueue of this engine to the scrub (hs_scrub_sig_cache): every tick then also audits the next
        buckets_per_tick buckets of its signature cache (VerifyQueue.sig_audit), wrapping around, and a tick that corrected an entry
        calls back with AUDIT_SIGCACHE in found.  None detaches."""
        self._check(self.lib.hs_scrub_sig_cache(self.h, queue.h if queue is not None else None, int(buckets_per_tick)), "hs_scrub_sig_cache")

    def explain(self, recs):
        """Table-free re-check of (n,128) uint8 records (hs_explain_rec128) -> uint8[n] of WHY_* bits, one per failed check.  The strict
        verdict is 1 iff the byte is 0; the batch-eq verdict is 1 iff it has no bit outside WHY_A_SMALL | WHY_R_SMALL."""
        recs = _u8(recs, 128).reshape(-1, 128)
        n = recs.shape[0]
        why = np.zeros(max(1, n), dtype=np.uint8)
        self._check(self.lib.hs_explain_rec128(self.h, _ptr(recs), n, _ptr(why)), "hs_explain_rec128")
        return why[:n]

    @property
    def last_error(self):
        return self.lib.hs_last_error(self.h).decode()

    # ---- host-buffer API -------------------------------------------------------------------------------------
    def verify_rec128(self, recs, mode=MODE_STRICT):
        """recs: (n,128) uint8 [sig64|pk32|msg32] -> bool[n]"""
        return _verify_rec128(self, self.lib.hs_verify_rec128, "hs_verify_rec128", recs, mode)

    def verify_strict_batch(self, recs):
        recs = _u8(recs, 128).reshape(-1, 128)
        n = recs.shape[0]
        bm = np.zeros((n + 31) // 32, dtype=np.uint32)
        self._check(self.lib.hs_verify_strict_batch(self.h, _ptr(recs), n, _ptr(bm)), "hs_verify_strict_batch")
        return bitmap_to_bools(bm, n)

    def verify_var(self, sig, pk, msgs, off, mode=MODE_STRICT):
        sig = _u8(sig, 64).reshape(-1, 64)
        pk = _u8(pk, 32).reshape(-1, 32)
        n = sig.shape[0]
        off = np.ascontiguousarray(off, dtype=np.uint64)
        assert pk.shape[0] == n and off.shape[0] == n + 1
        msgs = _u8(msgs)
        bm = np.zeros((n + 31) // 32, dtype=np.uint32)
        self._check(self.lib.hs_verify_var(self.h, _ptr(sig), _ptr(pk), _ptr(msgs) if msgs.size else None, _ptr(off), n, mode, _ptr(bm)),
                    "hs_verify_var")
        return bitmap_to_bools(bm, n)

    def verify_batch_shared_msg(self, digest, votes, want_bitmap=False):
        """votes: (n,96) uint8 [pk32|sig64].  Returns all_ok (and bool[n] when want_bitmap)."""
        digest = _u8(digest)
        assert digest.size == 32
        votes = _u8(votes, 96).reshape(-1, 96)
        n = votes.shape[0]
        ok = ctypes.c_int(0)
        bm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32) if want_bitmap else None
        self._check(self.lib.hs_verify_batch_shared_msg(self.h, _ptr(digest), _ptr(votes) if n else None, n, ctypes.byref(ok), _ptr(bm)),
                    "hs_verify_batch_shared_msg")
        return (bool(ok.value), bitmap_to_bools(bm, n)) if want_bitmap else bool(ok.value)

    def verify_qcs(self, preimages, sig, qc_idx, pk=None, validator_idx=None, want_votes=False):
        """Many QCs in one pass: preimages (n_qc,40) = hash||round_le; vote i -> certificate qc_idx[i].  Returns bool[n_qc]
        (and bool[n_votes] when want_votes)."""
        pre = _u8(preimages, 40).reshape(-1, 40)
        sig = _u8(sig, 64).reshape(-1, 64)
        n_qc, n = pre.shape[0], sig.shape[0]
        qi = np.ascontiguousarray(qc_idx, dtype=np.uint32)
        assert qi.shape[0] == n and (pk is None) != (validator_idx is None)
        pk = None if pk is None else _u8(pk, 32).reshape(-1, 32)
        vidx = None if validator_idx is None else np.ascontiguousarray(validator_idx, dtype=np.uint32)
        qbm = np.zeros(max(1, (n_qc + 31) // 32), dtype=np.uint32)
        vbm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32) if want_votes else None
        self._check(self.lib.hs_verify_qcs(self.h, _ptr(pre) if n_qc else None, n_qc, _ptr(pk), _ptr(vidx), _ptr(sig) if n else None,
                                           _ptr(qi) if n else None, n, _ptr(vbm), _ptr(qbm)), "hs_verify_qcs")
        out = bitmap_to_bools(qbm, n_qc)
        return (out, bitmap_to_bools(vbm, n)) if want_votes else out

    def verify_tcs(self, tc_rounds, sig, high_qc_rounds, tc_idx=None, pk=None, validator_idx=None, want_votes=False):
        """TC::verify for many TCs (tc_idx given) or Timeout signatures (tc_idx None: one vote per certificate): the 16-byte
        digests are built on the GPU from (tc_round, high_qc_round).  Returns bool[n_tc] (and bool[n_votes])."""
        tr = np.ascontiguousarray(tc_rounds, dtype=np.uint64)
        hq = np.ascontiguousarray(high_qc_rounds, dtype=np.uint64)
        sig = _u8(sig, 64).reshape(-1, 64)
        n, n_tc = sig.shape[0], tr.shape[0]
        assert hq.shape[0] == n and (pk is None) != (validator_idx is None)
        ti = None if tc_idx is None else np.ascontiguousarray(tc_idx, dtype=np.uint32)
        pk = None if pk is None else _u8(pk, 32).reshape(-1, 32)
        vidx = None if validator_idx is None else np.ascontiguousarray(validator_idx, dtype=np.uint32)
        tbm = np.zeros(max(1, (n_tc + 31) // 32), dtype=np.uint32)
        vbm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32) if want_votes else None
        self._check(self.lib.hs_verify_tcs(self.h, _ptr(tr) if n_tc else None, n_tc, _ptr(pk), _ptr(vidx), _ptr(sig) if n else None, _ptr(hq) if n else None,
                                           _ptr(ti), n, _ptr(vbm), _ptr(tbm)), "hs_verify_tcs")
        out = bitmap_to_bools(tbm, n_tc)
        return (out, bitmap_to_bools(vbm, n)) if want_votes else out

    def verify_groups(self, preimages, pre_off, sig, msg_idx, group_idx, n_groups, mode=None, pk=None, validator_idx=None, want_items=False):
        """hs_verify_groups: items over GPU-hashed variable-length preimages, per-item verdict mode, per-group AND."""
        return _verify_groups(self, self.lib.hs_verify_groups, "hs_verify_groups", preimages, pre_off, sig, msg_idx, group_idx, n_groups, mode, pk,
                              validator_idx, want_items)

    def keygen_batch(self, seeds):
        """RFC 8032 public keys of n 32-byte seeds, computed on the GPU (load generation; hs_keygen_batch)."""
        seeds = _u8(seeds, 32).reshape(-1, 32)
        out = np.zeros_like(seeds)
        self._check(self.lib.hs_keygen_batch(self.h, _ptr(seeds), seeds.shape[0], _ptr(out)), "hs_keygen_batch")
        return out

    def sign_digests(self, seeds, pks, digests, key_idx=None):
        """RFC 8032 signatures over 32-byte digests, made on the GPU (load generation; hs_sign_digests)."""
        seeds = _u8(seeds, 32).reshape(-1, 32)
        pks = _u8(pks, 32).reshape(-1, 32)
        digests = _u8(digests, 32).reshape(-1, 32)
        ki = None if key_idx is None else np.ascontiguousarray(key_idx, dtype=np.uint32)
        n = digests.shape[0]
        out = np.zeros((n, 64), dtype=np.uint8)
        self._check(self.lib.hs_sign_digests(self.h, _ptr(seeds), _ptr(pks), seeds.shape[0], _ptr(ki), _ptr(digests), n, _ptr(out)), "hs_sign_digests")
        return out

    def committee_register(self, pks):
        return _committee_register(self, self.lib.hs_committee_register, "hs_committee_register", pks)

    def committee_update(self, add=None, remove=None):
        """Incremental epoch change (hs_committee_update): returns the indices assigned to the added keys."""
        return _committee_update(self, self.lib.hs_committee_update, "hs_committee_update", add, remove)

    def committee_stage(self, add=None, remove=None):
        """Prepares a committee change off the verify path (hs_committee_stage): returns the indices the added keys will have.  Nothing
        changes for verification until committee_commit; stage + commit leaves the engine as update(add) then update(remove=remove)."""
        return _committee_update(self, self.lib.hs_committee_stage, "hs_committee_stage", add, remove)

    def committee_stage_register(self, pks, key_bits=0):
        """Builds and proves a whole new key store for pks beside the live one (hs_committee_stage_register): returns the keys' validity
        (bool[N]) and the window.  Nothing changes for verification until committee_commit; stage + commit leaves the engine as
        committee_register(pks) at that window.  key_bits 0: the widest window that fits beside the live store; 8..17: that window."""
        pks = _u8(pks, 32).reshape(-1, 32)
        n = pks.shape[0]
        bm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32)
        bits = ctypes.c_int(0)
        self._check(self.lib.hs_committee_stage_register(self.h, _ptr(pks) if n else None, n, int(key_bits), _ptr(bm), ctypes.byref(bits)),
                    "hs_committee_stage_register")
        self._staged_keys = n
        return bitmap_to_bools(bm, n), bits.value

    def committee_commit(self):
        """Switches the staged change in (hs_committee_commit): builds no table.  A staged registration replaces the committee."""
        self._check(self.lib.hs_committee_commit(self.h), "hs_committee_commit")
        if getattr(self, "_staged_keys", None) is not None:
            self.n_keys, self._staged_keys = self._staged_keys, None

    def committee_discard(self):
        """Frees the staged slots or the staged store (hs_committee_discard); a no-op when nothing is staged."""
        self._check(self.lib.hs_committee_discard(self.h), "hs_committee_discard")
        self._staged_keys = None

    def set_table_budget(self, nbytes):
        self._check(self.lib.hs_set_table_budget(self.h, int(nbytes)), "hs_set_table_budget")

    def verify_committee(self, validator_idx, sig, digests, msg_idx=None, mode=MODE_STRICT):
        vidx = np.ascontiguousarray(validator_idx, dtype=np.uint32)
        sig = _u8(sig, 64).reshape(-1, 64)
        digests = _u8(digests, 32).reshape(-1, 32)
        n = sig.shape[0]
        assert vidx.shape[0] == n
        midx = None if msg_idx is None else np.ascontiguousarray(msg_idx, dtype=np.uint32)
        bm = np.zeros((n + 31) // 32, dtype=np.uint32)
        self._check(self.lib.hs_verify_committee(self.h, _ptr(vidx), _ptr(sig), _ptr(midx), _ptr(digests), digests.shape[0], n, mode, _ptr(bm)),
                    "hs_verify_committee")
        return bitmap_to_bools(bm, n)

    def digest32_batch(self, data, off):
        data = _u8(data)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        n = off.shape[0] - 1
        out = np.zeros((n, 32), dtype=np.uint8)
        self._check(self.lib.hs_digest32_batch(self.h, _ptr(data) if data.size else None, _ptr(off), n, _ptr(out)), "hs_digest32_batch")
        return out

    def verify_msgs(self, sig, msgs, msg_len, pk=None, validator_idx=None, mode=MODE_STRICT):
        """Reference-shaped call: verdict_i = Signature::verify(Digest(msg_i), key_i); msgs = n fixed-size messages."""
        return _verify_msgs(self, self.lib.hs_verify_msgs, "hs_verify_msgs", sig, msgs, msg_len, pk, validator_idx, mode)

    # ---- device-resident API (torch tensors on this engine's device; enqueued on torch's current stream) -------
    @staticmethod
    def _stream():
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def verify_rec128_dev(self, d_recs, d_bitmap, n, mode=MODE_STRICT):
        self._check(self.lib.hs_verify_rec128_dev(self.h, d_recs.data_ptr(), n, mode, d_bitmap.data_ptr(), self._stream()), "hs_verify_rec128_dev")

    def verify_var_dev(self, d_sig, d_pk, d_msgs, d_off, d_bitmap, n, mode=MODE_STRICT):
        self._check(self.lib.hs_verify_var_dev(self.h, d_sig.data_ptr(), d_pk.data_ptr(), d_msgs.data_ptr(), d_off.data_ptr(), n, mode,
                                               d_bitmap.data_ptr(), self._stream()), "hs_verify_var_dev")

    def verify_committee_dev(self, d_vidx, d_sig, d_digests, d_bitmap, n, d_midx=None, mode=MODE_STRICT):
        self._check(self.lib.hs_verify_committee_dev(self.h, d_vidx.data_ptr(), d_sig.data_ptr(), None if d_midx is None else d_midx.data_ptr(),
                                                     d_digests.data_ptr(), n, mode, d_bitmap.data_ptr(), self._stream()),
                    "hs_verify_committee_dev")

    def verify_msgs_dev(self, d_sig, d_msgs, msg_len, d_digests, d_bitmap, n, d_pk=None, d_vidx=None, mode=MODE_STRICT):
        self._check(self.lib.hs_verify_msgs_dev(self.h, d_sig.data_ptr(), None if d_pk is None else d_pk.data_ptr(),
                                                None if d_vidx is None else d_vidx.data_ptr(), d_msgs.data_ptr(), msg_len, n, mode,
                                                d_digests.data_ptr(), d_bitmap.data_ptr(), self._stream()), "hs_verify_msgs_dev")

    def verify_qc_votes_dev(self, d_qc_digests, d_sig, d_qc_idx, d_vote_bitmap, n, d_pk=None, d_vidx=None):
        self._check(self.lib.hs_verify_qc_votes_dev(self.h, d_qc_digests.data_ptr(), None if d_pk is None else d_pk.data_ptr(),
                                                    None if d_vidx is None else d_vidx.data_ptr(), d_sig.data_ptr(), d_qc_idx.data_ptr(), n,
                                                    d_vote_bitmap.data_ptr(), self._stream()), "hs_verify_qc_votes_dev")

    def qc_and_dev(self, d_vote_bitmap, d_qc_idx, n_votes, n_qc, d_qc_bitmap):
        self._check(self.lib.hs_qc_and_dev(self.h, d_vote_bitmap.data_ptr(), d_qc_idx.data_ptr(), n_votes, n_qc, d_qc_bitmap.data_ptr(), self._stream()),
                    "hs_qc_and_dev")

    def verify_groups_dev(self, d_pre, d_off, n_msgs, d_sig, d_msg_idx, d_item_bitmap, n_items, d_mode=None, d_pk=None, d_vidx=None):
        """hs_verify_groups_dev: verify_groups with device arrays, enqueued on torch's current stream.  d_item_bitmap receives each item's
        verdict in its own mode (d_mode None = all strict); group verdicts: qc_and_dev(d_item_bitmap, d_group_idx, n_items, n_groups, ..)."""
        ptr = lambda t: None if t is None else t.data_ptr()
        self._check(self.lib.hs_verify_groups_dev(self.h, ptr(d_pre), ptr(d_off), n_msgs, ptr(d_sig), ptr(d_pk), ptr(d_vidx), ptr(d_msg_idx),
                                                  ptr(d_mode), n_items, ptr(d_item_bitmap), self._stream()), "hs_verify_groups_dev")

    def explain_groups_dev(self, d_pre, d_off, n_msgs, d_sig, d_pk, d_msg_idx, d_item_bitmap, n_items, d_why, d_out, d_mode=None,
                           max_explain=0):
        """hs_explain_groups_dev: the table-free re-check of Engine.explain for the items of a verify_groups_dev pass whose bit in
        d_item_bitmap is 0 (the lowest-index max_explain of them; 0 = all), enqueued on torch's current stream.  d_pk holds key bytes
        (for a committee-indexed pass, the caller's map gathered by validator index).  d_why (uint8, n_items) receives each examined
        item's WHY_* mask and WHY_NOT_EXAMINED elsewhere; d_out (int32 / uint32, EXPLAIN_DEV_OUT) receives the items whose bit is 0, the
        items examined, the engine faults among them (rejected, yet valid in their mode) and the lowest faulting index (0xffffffff: none)."""
        ptr = lambda t: None if t is None else t.data_ptr()
        self._check(self.lib.hs_explain_groups_dev(self.h, ptr(d_pre), ptr(d_off), n_msgs, ptr(d_sig), ptr(d_pk), ptr(d_msg_idx), ptr(d_mode),
                                                   ptr(d_item_bitmap), n_items, max_explain, ptr(d_why), ptr(d_out), self._stream()),
                    "hs_explain_groups_dev")

    def keygen_batch_dev(self, d_seeds, d_pks, n):
        self._check(self.lib.hs_keygen_batch_dev(self.h, d_seeds.data_ptr(), n, d_pks.data_ptr(), self._stream()), "hs_keygen_batch_dev")

    def sign_digests_dev(self, d_seeds, d_pks, n_keys, d_digests, d_sig, n, d_key_idx=None):
        self._check(self.lib.hs_sign_digests_dev(self.h, d_seeds.data_ptr(), d_pks.data_ptr(), n_keys, None if d_key_idx is None else d_key_idx.data_ptr(),
                                                 d_digests.data_ptr(), n, d_sig.data_ptr(), self._stream()), "hs_sign_digests_dev")

    def set_deferred(self, on):
        """Deferred-results mode for streams of `_dev` passes (hs_set_deferred): call results_wait() before reading bitmaps."""
        self._check(self.lib.hs_set_deferred(self.h, 1 if on else 0), "hs_set_deferred")

    def results_wait(self):
        self._check(self.lib.hs_results_wait(self.h, self._stream()), "hs_results_wait")

    def digest32_fixed_dev(self, d_msgs, msg_len, d_out, n):
        self._check(self.lib.hs_digest32_fixed_dev(self.h, d_msgs.data_ptr(), msg_len, n, d_out.data_ptr(), self._stream()), "hs_digest32_fixed_dev")

    def digest32_dev(self, d_data, d_off, d_out, n):
        self._check(self.lib.hs_digest32_dev(self.h, d_data.data_ptr(), d_off.data_ptr(), n, d_out.data_ptr(), self._stream()), "hs_digest32_dev")


# Marshalling of the host-pointer calls that Engine and MultiEngine both make: fn is the C entry point, owner.h its handle and
# owner._check its error check.
def _verify_rec128(owner, fn, name, recs, mode):
    recs = _u8(recs, 128).reshape(-1, 128)
    n = recs.shape[0]
    bm = np.zeros((n + 31) // 32, dtype=np.uint32)
    owner._check(fn(owner.h, _ptr(recs), n, mode, _ptr(bm)), name)
    return bitmap_to_bools(bm, n)


def _verify_msgs(owner, fn, name, sig, msgs, msg_len, pk, validator_idx, mode):
    sig = _u8(sig, 64).reshape(-1, 64)
    n = sig.shape[0]
    msgs = _u8(msgs)
    assert msgs.size == n * msg_len and (pk is None) != (validator_idx is None)
    pk = None if pk is None else _u8(pk, 32).reshape(-1, 32)
    vidx = None if validator_idx is None else np.ascontiguousarray(validator_idx, dtype=np.uint32)
    bm = np.zeros((n + 31) // 32, dtype=np.uint32)
    owner._check(fn(owner.h, _ptr(sig), _ptr(pk), _ptr(vidx), _ptr(msgs), msg_len, n, mode, _ptr(bm)), name)
    return bitmap_to_bools(bm, n)


def _verify_groups(owner, fn, name, preimages, pre_off, sig, msg_idx, group_idx, n_groups, mode, pk, validator_idx, want_items):
    pre = _u8(preimages)
    off = np.ascontiguousarray(pre_off, dtype=np.uint64)
    sig = _u8(sig, 64).reshape(-1, 64)
    n = sig.shape[0]
    mi = np.ascontiguousarray(msg_idx, dtype=np.uint32)
    gi = np.ascontiguousarray(group_idx, dtype=np.uint32)
    mo = None if mode is None else np.ascontiguousarray(mode, dtype=np.uint8)
    assert (pk is None) != (validator_idx is None) and mi.shape[0] == n == gi.shape[0]
    pk = None if pk is None else _u8(pk, 32).reshape(-1, 32)
    vidx = None if validator_idx is None else np.ascontiguousarray(validator_idx, dtype=np.uint32)
    gbm = np.zeros(max(1, (n_groups + 31) // 32), dtype=np.uint32)
    ibm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32) if want_items else None
    owner._check(fn(owner.h, _ptr(pre) if pre.size else None, _ptr(off), off.shape[0] - 1, _ptr(sig) if n else None, _ptr(pk), _ptr(vidx),
                    _ptr(mi) if n else None, _ptr(gi) if n else None, _ptr(mo), n, n_groups, _ptr(ibm), _ptr(gbm)), name)
    out = bitmap_to_bools(gbm, n_groups)
    return (out, bitmap_to_bools(ibm, n)) if want_items else out


def _committee_register(owner, fn, name, pks):
    pks = _u8(pks, 32).reshape(-1, 32)
    n = pks.shape[0]
    bm = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32)
    owner._check(fn(owner.h, _ptr(pks) if n else None, n, _ptr(bm)), name)
    owner.n_keys = n
    owner._staged_keys = None  # a registration discards a staged one
    return bitmap_to_bools(bm, n)


def _committee_update(owner, fn, name, add, remove):
    add = np.zeros((0, 32), np.uint8) if add is None else _u8(add, 32).reshape(-1, 32)
    rem = np.zeros(0, np.uint32) if remove is None else np.ascontiguousarray(remove, dtype=np.uint32)
    out = np.zeros(max(1, add.shape[0]), dtype=np.uint32)
    owner._check(fn(owner.h, _ptr(add) if add.shape[0] else None, add.shape[0], _ptr(rem) if rem.shape[0] else None, rem.shape[0], _ptr(out)), name)
    owner._staged_keys = None  # an update discards a staged registration; an incremental stage succeeds only with none pending
    return out[: add.shape[0]]


class MultiEngine:
    """Python handle on one hs_multi: several member contexts in this process (include/hs_crypto.h, hs_multi_*).  A host-pointer verify
    call of at least HS_MULTI_MIN_SHARD records per member is sharded across the members; a smaller one runs whole on one member, chosen
    round-robin.  Verdicts equal the same Engine call bit for bit.  devices may list a device more than once."""

    MIN_SHARD = 4096  # HS_MULTI_MIN_SHARD

    def __init__(self, devices, base_window=0, key_window=0, key_cache=True):
        self.lib = _lib.load()
        devs = np.ascontiguousarray([int(d) for d in devices], dtype=np.int32)
        h = ctypes.c_void_p()
        flags = (int(base_window) & 0xff) | ((int(key_window) & 0xff) << 8) | (0 if key_cache else 0x10000)
        rc = self.lib.hs_multi_create(ctypes.byref(h), _ptr(devs) if devs.size else None, devs.size, flags)
        if rc != 0 or not h:
            raise EngineError("hs_multi_create(devices=%s) failed with status %d (no GPU / bad ordinal / CUDA error); there is no CPU fallback"
                              % (list(devs), rc))
        self.h = h
        self.devices = [int(d) for d in devs]
        self.n_keys = 0
        self._members = [Engine._view(self.lib, self.lib.hs_multi_member(h, i), d) for i, d in enumerate(self.devices)]

    def member(self, i):
        """Member i as a non-owning Engine: every single-device call works on it.  Do not change its committee directly."""
        return self._members[i]

    def __len__(self):
        return len(self._members)

    def close(self):
        """Closes the queues created on the members, then destroys the members and joins the worker threads."""
        for e in getattr(self, "_members", []):
            e.close()
        if getattr(self, "h", None):
            self.lib.hs_multi_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed: status %d: %s" % (what, rc, self.lib.hs_multi_last_error(self.h).decode()))

    @property
    def last_error(self):
        return self.lib.hs_multi_last_error(self.h).decode()

    def register_committee(self, pks):
        """hs_multi_committee_register: the same committee on every member; returns the keys' validity (bool[N])."""
        return _committee_register(self, self.lib.hs_multi_committee_register, "hs_multi_committee_register", pks)

    def update_committee(self, add=None, remove=None):
        """hs_multi_committee_update: returns the indices assigned to the added keys (the same on every member)."""
        return _committee_update(self, self.lib.hs_multi_committee_update, "hs_multi_committee_update", add, remove)

    def stage_committee(self, add=None, remove=None):
        """The staged committee change on every member, member by member through hs_committee_stage (as a repair is): stages on every
        member at once, one thread each, and returns the indices, the same on every member.  If any member fails, or the members
        return different indices, the stage is discarded on every member and EngineError raised: nothing stays staged."""
        res = [None] * len(self._members)

        def stage(i):
            try:
                res[i] = self._members[i].committee_stage(add, remove)
            except EngineError as e:
                res[i] = e

        threads = [threading.Thread(target=stage, args=(i,)) for i in range(len(self._members))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        err = next((r for r in res if isinstance(r, EngineError)), None)
        if err is None and any(not np.array_equal(r, res[0]) for r in res[1:]):
            err = EngineError("stage_committee: the members gave different indices")
        if err is not None:
            self.discard_committee()
            raise err
        self._staged_keys = None
        return res[0]

    def stage_register_committee(self, pks, key_bits=0):
        """The staged registration on every member, member by member through hs_committee_stage_register: stages on every member at
        once, one thread each, and returns the keys' validity (bool[N]) and the window, the same on every member.  If any member fails,
        or the members differ in either, the stage is discarded on every member and EngineError raised: every member keeps its committee.
        commit_committee switches it in."""
        res = [None] * len(self._members)

        def stage(i):
            try:
                res[i] = self._members[i].committee_stage_register(pks, key_bits)
            except EngineError as e:
                res[i] = e

        threads = [threading.Thread(target=stage, args=(i,)) for i in range(len(self._members))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        err = next((r for r in res if isinstance(r, EngineError)), None)
        if err is None and any(not np.array_equal(r[0], res[0][0]) or r[1] != res[0][1] for r in res[1:]):
            err = EngineError("stage_register_committee: the members gave different validity or windows")
        if err is not None:
            self.discard_committee()
            raise err
        self._staged_keys = len(res[0][0])
        return res[0]

    def commit_committee(self):
        """hs_committee_commit on every member.  After a failure the members may differ: re-register."""
        for e in self._members:
            e.committee_commit()
        if getattr(self, "_staged_keys", None) is not None:
            self.n_keys, self._staged_keys = self._staged_keys, None

    def discard_committee(self):
        """hs_committee_discard on every member."""
        for e in self._members:
            e.committee_discard()
        self._staged_keys = None

    def verify_rec128(self, recs, mode=MODE_STRICT):
        return _verify_rec128(self, self.lib.hs_multi_verify_rec128, "hs_multi_verify_rec128", recs, mode)

    def verify_msgs(self, sig, msgs, msg_len, pk=None, validator_idx=None, mode=MODE_STRICT):
        return _verify_msgs(self, self.lib.hs_multi_verify_msgs, "hs_multi_verify_msgs", sig, msgs, msg_len, pk, validator_idx, mode)

    def verify_groups(self, preimages, pre_off, sig, msg_idx, group_idx, n_groups, mode=None, pk=None, validator_idx=None, want_items=False):
        return _verify_groups(self, self.lib.hs_multi_verify_groups, "hs_multi_verify_groups", preimages, pre_off, sig, msg_idx, group_idx, n_groups,
                              mode, pk, validator_idx, want_items)


class _WhyCount(int):
    """The record count of an explain ticket: its words hold one why byte per record, four to a word."""


class VerifyQueue:
    """hs_queue_* (include/hs_crypto.h): submit 1..64 records (submit) or a whole certificate (submit_group, or submit_msgs with the
    signed preimages instead of their Digests) without blocking;
    a dispatcher thread coalesces whatever is pending into one latency-path launch.  Verdicts equal Engine.verify_rec128 on the
    same records (per record and its mode for a group).  A ticket is read once:
    by poll() / wait(), or by the callback given to submit() (called on the queue's thread as callback(ticket, status, bools);
    status != 0 means engine failure: reject every signature)."""

    def __init__(self, engine, ring_records=0):
        self.engine = engine
        self.lib = engine.lib
        h = ctypes.c_void_p()
        engine._check(self.lib.hs_queue_create(engine.h, int(ring_records), ctypes.byref(h)), "hs_queue_create")
        self.h = h
        self._lock = threading.Lock()
        self._n = {}          # ticket -> records, for tickets read by poll / wait
        self._callbacks = {}  # user id -> (callback, records)
        self._next_id = 1
        self._trampoline = _lib.QUEUE_CB(self._on_done)  # one C callback for the queue's lifetime
        engine._queues.append(self)

    def _on_done(self, user, ticket, status, bitmap):
        with self._lock:
            fn, n = self._callbacks.pop(user)
        words = np.ctypeslib.as_array(bitmap, shape=(self._n_words(n),)).copy()
        fn(int(ticket), int(status), self._bools(words, n))

    @staticmethod
    def _n_words(n):
        """Words of a ticket's verdict bitmap: n is a record count, or (n_groups, n_items) for a batch ticket (the why bytes of an
        explain ticket: (n + 3) / 4 words)."""
        if isinstance(n, _WhyCount):
            return (n + 3) // 4
        return (n[0] + 31) // 32 + (n[1] + 31) // 32 if isinstance(n, tuple) else (n + 31) // 32

    @staticmethod
    def _bools(words, n):
        if isinstance(n, _WhyCount):  # an explain ticket: one HS_WHY_* byte per record
            return words.view(np.uint8)[:n].copy()
        if isinstance(n, tuple):  # a batch ticket: group words, then item words
            gw = (n[0] + 31) // 32
            return bitmap_to_bools(words[:gw], n[0]), bitmap_to_bools(words[gw:], n[1])
        return bitmap_to_bools(words, n)

    def submit(self, recs, mode=MODE_STRICT, callback=None):
        """recs: (n,128) uint8 [sig64|pk32|msg32], 1 <= n <= 64.  Returns the ticket, or None when the ring is full (retry later)."""
        return self._submit(self.lib.hs_queue_submit, "hs_queue_submit", recs, mode, callback)

    def submit_group(self, recs, modes=None, callback=None):
        """One consensus message's whole certificate (a Block: author strict + QC votes batch-eq + TC votes strict; a Timeout with
        its high_qc; a TC; a QC) as ONE request.  recs: (n,128) uint8, 1 <= n <= the ring's capacity; modes: uint8[n] of MODE_*
        per record (None = all strict).  Returns the ticket, or None when the ring has no room now (verify synchronously)."""
        recs = _u8(recs, 128).reshape(-1, 128)
        if modes is not None:
            modes = np.ascontiguousarray(modes, dtype=np.uint8).reshape(-1)
            if modes.shape[0] != recs.shape[0]:
                raise ValueError("submit_group: %d modes for %d records" % (modes.shape[0], recs.shape[0]))
        return self._submit(self.lib.hs_queue_submit_group, "hs_queue_submit_group", recs, None if modes is None else _ptr(modes), callback)

    def submit_msgs(self, preimages, pre_off, sig, pk, msg_idx, modes=None, callback=None):
        """One consensus message's signatures as ONE request with the signed preimages instead of their Digests (hs_queue_submit_msgs):
        record i is (sig[i], pk[i]) over SHA-512(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]))[..32], hashed on the
        GPU, judged by modes[i] (None = all strict) — the arrays wire.ingest_frames returns for one frame.  Returns the ticket, or None
        when the ring or the preimage arena has no room now (verify synchronously)."""
        pre = _u8(preimages)
        off = np.ascontiguousarray(pre_off, dtype=np.uint64).reshape(-1)
        sig = _u8(sig, 64).reshape(-1, 64)
        pk = _u8(pk, 32).reshape(-1, 32)
        mi = np.ascontiguousarray(msg_idx, dtype=np.uint32).reshape(-1)
        n = sig.shape[0]
        mo = None if modes is None else np.ascontiguousarray(modes, dtype=np.uint8).reshape(-1)
        if pk.shape[0] != n or mi.shape[0] != n or (mo is not None and mo.shape[0] != n) or off.shape[0] < 1:
            raise ValueError("submit_msgs: %d signatures, %d keys, %d message indices, %s modes, %d offsets"
                             % (n, pk.shape[0], mi.shape[0], "no" if mo is None else mo.shape[0], off.shape[0]))
        return self._enqueue("hs_queue_submit_msgs", n, callback, lambda cb, user, t: self.lib.hs_queue_submit_msgs(
            self.h, _ptr(pre) if pre.size else None, _ptr(off), off.shape[0] - 1, _ptr(sig) if n else None, _ptr(pk) if n else None,
            _ptr(mi) if n else None, _ptr(mo), n, cb, user, t))

    def batch(self, max_items, max_bytes):
        """Turns the batch lane on (hs_queue_batch): submit_batch requests of up to max_items items and max_bytes of arena region each.
        (0, 0) turns it off (the default).  Resizing or turning it off first waits for every batch request already submitted."""
        self.engine._check(self.lib.hs_queue_batch(self.h, int(max_items), int(max_bytes)), "hs_queue_batch")

    def submit_batch(self, preimages, pre_off, sig, pk, msg_idx, group_idx, n_groups, modes=None, callback=None):
        """Engine.verify_groups (with key bytes) as ONE non-blocking request on the batch lane (hs_queue_submit_batch): item i is
        (sig[i], pk[i]) over SHA-512(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]))[..32] in group group_idx[i], judged by
        modes[i] (None = all strict).  poll / wait / the callback give (group bools, item bools), equal to verify_groups on the same
        arrays.  Returns the ticket, or None when the lane's arena has no room now."""
        pre = _u8(preimages)
        off = np.ascontiguousarray(pre_off, dtype=np.uint64).reshape(-1)
        sig = _u8(sig, 64).reshape(-1, 64)
        pk = _u8(pk, 32).reshape(-1, 32)
        mi = np.ascontiguousarray(msg_idx, dtype=np.uint32).reshape(-1)
        gi = np.ascontiguousarray(group_idx, dtype=np.uint32).reshape(-1)
        n = sig.shape[0]
        mo = None if modes is None else np.ascontiguousarray(modes, dtype=np.uint8).reshape(-1)
        if pk.shape[0] != n or mi.shape[0] != n or gi.shape[0] != n or (mo is not None and mo.shape[0] != n) or off.shape[0] < 1:
            raise ValueError("submit_batch: %d signatures, %d keys, %d message indices, %d group indices, %s modes, %d offsets"
                             % (n, pk.shape[0], mi.shape[0], gi.shape[0], "no" if mo is None else mo.shape[0], off.shape[0]))
        return self._enqueue("hs_queue_submit_batch", (int(n_groups), n), callback, lambda cb, user, t: self.lib.hs_queue_submit_batch(
            self.h, _ptr(pre) if pre.size else None, _ptr(off), off.shape[0] - 1, _ptr(sig) if n else None, _ptr(pk) if n else None,
            _ptr(mi) if n else None, _ptr(gi) if n else None, _ptr(mo), n, int(n_groups), cb, user, t))

    BATCH_STATS = ("passes", "items", "groups", "preimage_bytes", "outside_committee")

    def batch_stats(self):
        """Counters of completed batch passes (hs_queue_batch_stats): passes, items, groups, preimage bytes hashed, and items whose
        key was outside the committee (every item when none is registered)."""
        out = (ctypes.c_uint64 * len(self.BATCH_STATS))()
        self.engine._check(self.lib.hs_queue_batch_stats(self.h, out), "hs_queue_batch_stats")
        return dict(zip(self.BATCH_STATS, (int(x) for x in out)))

    def explain(self, max_records, max_bytes):
        """Turns the explain lane on (hs_queue_explain): submit_explain / submit_explain_msgs requests of up to max_records records and
        max_bytes of arena region each.  (0, 0) turns it off (the default).  Resizing or turning it off first waits for every explain
        request already submitted."""
        self.engine._check(self.lib.hs_queue_explain(self.h, int(max_records), int(max_bytes)), "hs_queue_explain")

    def submit_explain(self, recs, callback=None):
        """Engine.explain as ONE non-blocking request on the explain lane (hs_queue_submit_explain).  recs: (n,128) uint8.  poll / wait /
        the callback give uint8[n] of HS_WHY_* masks, byte for byte those of Engine.explain.  Returns the ticket, or None when the lane's
        arena has no room now (back-pressure)."""
        recs = _u8(recs, 128).reshape(-1, 128)
        n = recs.shape[0]
        return self._enqueue("hs_queue_submit_explain", _WhyCount(n), callback,
                             lambda cb, user, t: self.lib.hs_queue_submit_explain(self.h, _ptr(recs) if n else None, n, cb, user, t))

    def submit_explain_msgs(self, preimages, pre_off, sig, pk, msg_idx, callback=None):
        """The same with the signed preimages instead of their Digests (hs_queue_submit_explain_msgs), in the arrays of submit_msgs
        without modes: record i is (sig[i], pk[i]) over SHA-512(preimages[pre_off[msg_idx[i]] .. pre_off[msg_idx[i] + 1]))[..32], hashed
        on the GPU.  Returns the ticket, or None when the lane's arena has no room now."""
        pre = _u8(preimages)
        off = np.ascontiguousarray(pre_off, dtype=np.uint64).reshape(-1)
        sig = _u8(sig, 64).reshape(-1, 64)
        pk = _u8(pk, 32).reshape(-1, 32)
        mi = np.ascontiguousarray(msg_idx, dtype=np.uint32).reshape(-1)
        n = sig.shape[0]
        if pk.shape[0] != n or mi.shape[0] != n or off.shape[0] < 1:
            raise ValueError("submit_explain_msgs: %d signatures, %d keys, %d message indices, %d offsets" % (n, pk.shape[0], mi.shape[0], off.shape[0]))
        return self._enqueue("hs_queue_submit_explain_msgs", _WhyCount(n), callback, lambda cb, user, t: self.lib.hs_queue_submit_explain_msgs(
            self.h, _ptr(pre) if pre.size else None, _ptr(off), off.shape[0] - 1, _ptr(sig) if n else None, _ptr(pk) if n else None,
            _ptr(mi) if n else None, n, cb, user, t))

    EXPLAIN_STATS = ("launches", "records", "requests")

    def explain_stats(self):
        """Counters of completed explain launches (hs_queue_explain_stats): k_queue_explain launches, the records they carried, and the
        requests."""
        out = (ctypes.c_uint64 * len(self.EXPLAIN_STATS))()
        self.engine._check(self.lib.hs_queue_explain_stats(self.h, out), "hs_queue_explain_stats")
        return dict(zip(self.EXPLAIN_STATS, (int(x) for x in out)))

    def _submit(self, fn, name, recs, mode_arg, callback):
        recs = _u8(recs, 128).reshape(-1, 128)
        n = recs.shape[0]
        return self._enqueue(name, n, callback, lambda cb, user, t: fn(self.h, _ptr(recs), n, mode_arg, cb, user, t))

    def _enqueue(self, name, n, callback, call):
        """call(callback pointer or None, user id or None, ticket out-pointer) -> status."""
        t = ctypes.c_size_t(0)
        if callback is None:
            with self._lock:  # registered first: poll / wait from another thread may race the return
                rc = call(None, None, ctypes.byref(t))
                if rc == 0:
                    self._n[t.value] = n
        else:
            with self._lock:
                uid = self._next_id
                self._next_id += 1
                self._callbacks[uid] = (callback, n)
            rc = call(ctypes.cast(self._trampoline, ctypes.c_void_p), uid, ctypes.byref(t))
            if rc != 0:
                with self._lock:
                    self._callbacks.pop(uid, None)
        if rc == 3:  # HS_ERR_NOMEM: back-pressure
            return None
        self.engine._check(rc, name)
        return t.value

    def _take(self, ticket, rc, words):
        with self._lock:
            n = self._n.pop(ticket, None)
        self.engine._check(rc, "hs_queue ticket %d" % ticket)
        return self._bools(words, n)

    def _words(self, ticket):
        """The verdict buffer of a ticket read by poll / wait: (n + 31) / 32 words (at least 2: an unknown ticket is an error)."""
        with self._lock:
            n = self._n.get(int(ticket), 64)
        return np.zeros(max(2, self._n_words(n)), dtype=np.uint32)

    def poll(self, ticket):
        """None while the request is in flight, else its verdicts (bool[n]; a batch ticket: (group bools, item bools); an explain
        ticket: uint8[n] of why masks); consumes the ticket."""
        done = ctypes.c_int(0)
        words = self._words(ticket)
        rc = self.lib.hs_queue_poll(self.h, int(ticket), ctypes.byref(done), _ptr(words))
        if rc == 0 and not done.value:
            return None
        return self._take(ticket, rc, words)

    def wait(self, ticket):
        """Blocks until the request is done; returns its verdicts (bool[n]; a batch ticket: (group bools, item bools); an explain
        ticket: uint8[n] of why masks) and consumes the ticket."""
        words = self._words(ticket)
        rc = self.lib.hs_queue_wait(self.h, int(ticket), _ptr(words))
        return self._take(ticket, rc, words)

    STATS = ("small_launches", "small_records", "bulk_launches", "bulk_records", "slow_requests", "slow_records")

    def stats(self):
        """Counters since the queue was created (hs_queue_stats): k_verify_small launches and the records they carried (riders
        included), k_verify_bulk launches and their records, slow-path requests and their records."""
        out = (ctypes.c_uint64 * len(self.STATS))()
        self.engine._check(self.lib.hs_queue_stats(self.h, out), "hs_queue_stats")
        return dict(zip(self.STATS, (int(x) for x in out)))

    DIGEST_STATS = ("digest_launches", "preimages", "preimage_bytes", "msgs_requests")

    def digest_stats(self):
        """Counters since the queue was created (hs_queue_digest_stats): k_queue_digests launches, the preimages and preimage bytes
        they hashed, and the submit_msgs requests."""
        out = (ctypes.c_uint64 * len(self.DIGEST_STATS))()
        self.engine._check(self.lib.hs_queue_digest_stats(self.h, out), "hs_queue_digest_stats")
        return dict(zip(self.DIGEST_STATS, (int(x) for x in out)))

    def cert_cache(self, max_bytes):
        """Turns the certificate cache on (hs_queue_cert_cache): keep up to max_bytes of verified certificates, so an identical QC in a
        later submit_group / submit_msgs request is answered without verifying it again, and one still in flight is joined instead of
        verified twice.  Verdicts do not change.  0 turns it off (the default)."""
        self.engine._check(self.lib.hs_queue_cert_cache(self.h, int(max_bytes)), "hs_queue_cert_cache")

    CERT_STATS = ("lookups", "hits", "joins", "records_answered", "inserted", "bytes_held")

    def cert_stats(self):
        """Counters of the certificate cache (hs_queue_cert_stats): spans looked up, cache hits, in-flight joins, records answered
        without verifying them, spans inserted, and the bytes held now."""
        out = (ctypes.c_uint64 * len(self.CERT_STATS))()
        self.engine._check(self.lib.hs_queue_cert_stats(self.h, out), "hs_queue_cert_stats")
        return dict(zip(self.CERT_STATS, (int(x) for x in out)))

    def sig_cache(self, entries):
        """Turns the signature cache on (hs_queue_sig_cache): a table in HBM of at least `entries` records the queue's kernels
        accepted, so a signature verified once (a Timeout's author vote, then the same vote in the TC) is a probe that hits instead
        of a verify.  Verdicts do not change.  Resizing starts from an empty table; 0 turns it off (the default)."""
        self.engine._check(self.lib.hs_queue_sig_cache(self.h, int(entries)), "hs_queue_sig_cache")

    SIG_STATS = ("probed", "hits", "inserts", "evictions", "entries_held")

    def sig_stats(self):
        """Counters of the signature cache over completed launches (hs_queue_sig_stats): records probed, hits, inserts, inserts
        that evicted a live entry, and the entries held now."""
        out = (ctypes.c_uint64 * len(self.SIG_STATS))()
        self.engine._check(self.lib.hs_queue_sig_stats(self.h, out), "hs_queue_sig_stats")
        return dict(zip(self.SIG_STATS, (int(x) for x in out)))

    def sig_share(self, on):
        """Shares the signature cache (hs_queue_sig_share) with the synchronous verify calls on the engine and with the batch lane:
        their committee passes answer records the table holds and insert the strict records they accept, so a TC or Block verified
        synchronously after its Timeouts came through the queue costs probes.  Needs the cache on; one queue per engine.  Verdicts do
        not change.  False turns it off (the default)."""
        self.engine._check(self.lib.hs_queue_sig_share(self.h, 1 if on else 0), "hs_queue_sig_share")

    SIG_SHARE_STATS = ("probed", "hits", "inserts", "evictions", "passes")

    def sig_share_stats(self):
        """Counters of the shared passes (hs_queue_sig_share_stats): records probed, hits, inserts, inserts that evicted a live
        entry, and the shared passes."""
        out = (ctypes.c_uint64 * len(self.SIG_SHARE_STATS))()
        self.engine._check(self.lib.hs_queue_sig_share_stats(self.h, out), "hs_queue_sig_share_stats")
        return dict(zip(self.SIG_SHARE_STATS, (int(x) for x in out)))

    SIG_AUDIT_OUT = ("held", "corrected", "skipped", "first_position", "first_stored", "first_derived", "first_why")

    def sig_audit(self, first_bucket=0, n_buckets=0):
        """Audits the signature cache (hs_queue_sig_audit): every held entry of buckets [first_bucket, first_bucket + n_buckets) (0: to
        the end of the table) is re-checked from its 128 bytes with the table-free re-check of Engine.explain, and a flag byte that
        disagrees is corrected.  Returns a dict keyed by SIG_AUDIT_OUT: entries held, corrected and skipped (being written), and the
        first correction's position (bucket * 4 + way; None: no correction), stored and derived flag bytes and WHY_* mask.  Raises
        EngineError when the cache is off or the range leaves the table."""
        out = (ctypes.c_uint64 * len(self.SIG_AUDIT_OUT))()
        self.engine._check(self.lib.hs_queue_sig_audit(self.h, int(first_bucket), int(n_buckets), out), "hs_queue_sig_audit")
        r = dict(zip(self.SIG_AUDIT_OUT, (int(x) for x in out)))
        if r["first_position"] == 2**64 - 1:
            r["first_position"] = None
        return r

    SIG_AUDIT_STATS = ("audits", "checked", "corrected", "skipped", "passes")

    def sig_audit_stats(self):
        """Counters over sig_audit calls and scrub slices (hs_queue_sig_audit_stats): audits, entries re-checked, corrected, skipped,
        and full passes of the table."""
        out = (ctypes.c_uint64 * len(self.SIG_AUDIT_STATS))()
        self.engine._check(self.lib.hs_queue_sig_audit_stats(self.h, out), "hs_queue_sig_audit_stats")
        return dict(zip(self.SIG_AUDIT_STATS, (int(x) for x in out)))

    def generic(self, on):
        """Turns the generic-key device path on or off (hs_queue_generic): with it on, a request with a key outside the registered
        committee (every request, when none is registered) is verified by a queue kernel on the GPU instead of synchronously on the
        dispatcher thread, so it no longer holds up the other requests.  Verdicts do not change.  Off (the default) drains the
        generic launches in flight."""
        self.engine._check(self.lib.hs_queue_generic(self.h, 1 if on else 0), "hs_queue_generic")

    GENERIC_STATS = ("launches", "records", "requests")

    def generic_stats(self):
        """Counters of the generic path (hs_queue_generic_stats): k_queue_generic launches, the records they carried, and the
        requests."""
        out = (ctypes.c_uint64 * len(self.GENERIC_STATS))()
        self.engine._check(self.lib.hs_queue_generic_stats(self.h, out), "hs_queue_generic_stats")
        return dict(zip(self.GENERIC_STATS, (int(x) for x in out)))

    def close(self):
        """Completes every request in flight (callbacks fire) and joins the dispatcher thread."""
        if getattr(self, "h", None):
            self.lib.hs_queue_destroy(self.h)
            self.h = None
            if self in self.engine._queues:
                self.engine._queues.remove(self)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
