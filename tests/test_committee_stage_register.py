"""hs_committee_stage_register + hs_committee_commit / hs_committee_discard: a whole new key store built and proved beside the live one,
switched in at the commit.

GPU: stage_register(P, w) + commit on one context equals hs_committee_register(P) at window w on another (validity, slots, windows,
clean audits, verdicts on every path, and the incremental calls after it); nothing changes for verification before the commit; the
window changes both ways; every error leaves the live committee verifying and auditing clean; a vote burst with the signature cache
shared runs across the stage and the commit; a multi-device stage that fails on one member is discarded on every member."""
import ctypes
import threading

import numpy as np
import pytest

from test_committee_stage import Node, _audit_clean, _bad_keys, _by_index, _every_path, _keys, _sign
from test_table_repair import POKE_TABLE, _engine, _entry_off, hooklib  # noqa: F401  (hooklib: the -DHS_TEST_HOOKS build, a fixture)

pytestmark = pytest.mark.gpu
HS_ERR_ARG, HS_ERR_NOMEM, HS_ERR_SELFTEST = 2, 3, 4
SMALL_ORDER = np.array([1] + [0] * 31, np.uint8)  # the identity's encoding: decompresses, small order


def _new_committee(oracle, n, seed):
    """n keys: two that do not decompress, one of small order and one duplicated key (index 40 repeats index 3)."""
    seeds, pks = _keys(oracle, n, seed)
    pks[[17, n - 5]] = _bad_keys(oracle, 2, seed + 1)
    pks[29] = SMALL_ORDER
    pks[40] = pks[3]
    seeds[40] = seeds[3]
    return seeds, pks


def _stage_register_raw(e, pks, key_bits=0):
    """The C call itself: status, validity words and window, with sentinels in the outputs."""
    pks = np.ascontiguousarray(pks, np.uint8)
    bm = np.full(max(1, (len(pks) + 31) // 32), 0xAAAAAAAA, np.uint32)
    bits = ctypes.c_int(-1)
    rc = e.lib.hs_committee_stage_register(e.h, pks.ctypes.data_as(ctypes.c_void_p) if len(pks) else None, len(pks), key_bits,
                                           bm.ctypes.data_as(ctypes.c_void_p), ctypes.byref(bits))
    return rc, bm, bits.value


def _verdicts_by_index(e, oracle, node, recs, vidx):
    got = e.verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(recs), dtype=np.uint32))
    assert np.array_equal(got, _by_index(oracle, node, recs, vidx))
    return got


@pytest.mark.parametrize("n,window", [(64, 12), (1000, 10)])
def test_stage_register_and_commit_equal_a_registration(oracle, n, window):
    from hotstuff_b200 import Engine
    oseeds, opks = _keys(oracle, 48, 600 + n)
    seeds, pks = _new_committee(oracle, n, 610 + n)
    e1, e2 = Engine(0, key_window=window), Engine(0, key_window=window)
    try:
        e1.committee_register(opks)  # the live committee the stage replaces
        valid1, bits = e1.committee_stage_register(pks, window)
        assert bits == window
        e1.committee_commit()
        valid2 = e2.committee_register(pks)
        assert np.array_equal(valid1, valid2) and np.array_equal(valid1, [oracle.decompress_ok(bytes(k)) for k in pks])
        assert not valid1[17] and not valid1[n - 5] and valid1[29]
        assert e1.key_slots == e2.key_slots == n and e1.window_bits == e2.window_bits
        node = Node(pks)
        _audit_clean(e1, node)
        _audit_clean(e2, node)
        ki = np.array(list(range(0, n, max(1, n // 60))) + [3, 40, 17, 29, n - 1] * 4, np.int64)
        ki = ki[(ki != 17) & (ki != n - 5) & (ki != 29)]  # keys with a secret: records over them
        recs, pre = _sign(oracle, seeds, pks, ki, 620 + n, with_preimages=True)
        vidx = ki.astype(np.uint32)
        vidx[-4:] = [17, 29, n - 5, 40]  # invalid, small-order and duplicated slots by index
        for e in (e1, e2):
            _every_path(e, oracle, node, recs, pre, vidx)
        # the incremental calls after it agree
        _, npks = _keys(oracle, 6, 630 + n)
        up = [e.committee_update(npks[:3], [5]) for e in (e1, e2)]
        assert np.array_equal(up[0], up[1])
        node.update(npks[:3], up[0], [5])
        idx = [e.committee_stage(npks[3:6], [6]) for e in (e1, e2)]
        assert np.array_equal(idx[0], idx[1])
        for e in (e1, e2):
            e.committee_commit()
        node.apply(npks[3:6], idx[0], [6])
        _audit_clean(e1, node)
        _audit_clean(e2, node)
    finally:
        e1.close()
        e2.close()


def test_nothing_changes_before_the_commit(oracle):
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 64, 640)
    nseeds, npks = _keys(oracle, 32, 641)
    e = Engine(0, key_window=12)
    try:
        e.committee_register(pks)
        node = Node(pks)
        P = np.concatenate([pks[32:], npks])  # half the old set, half new keys
        all_seeds, all_pks = np.concatenate([seeds, nseeds]), np.concatenate([pks, npks])
        ki = np.array(list(range(0, 96, 3)) * 2)
        recs = _sign(oracle, all_seeds, all_pks, ki, 642, corrupt=0.1)
        old_recs = _sign(oracle, seeds, pks, np.arange(64), 643, corrupt=0.1)
        vidx = np.arange(64, dtype=np.uint32)

        def observe():
            v = [e.verify_rec128(recs, mode=m) for m in (0, 1)]
            q = e.queue()
            try:
                for i in range(len(recs)):
                    q.wait(q.submit(recs[i:i + 1]))
                st = q.stats()
            finally:
                q.close()
            return v, st, _verdicts_by_index(e, oracle, node, old_recs, vidx), e.key_slots, e.window_bits

        before = observe()
        valid, bits = e.committee_stage_register(P, 12)
        assert valid.all() and bits == 12
        after = observe()
        assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0]))
        assert before[1] == after[1] and np.array_equal(before[2], after[2])
        assert before[3] == after[3] == 64 and tuple(before[4]) == tuple(after[4]) and after[4][0] == 12
        for m in (0, 1):  # the new keys are on the generic path with the oracle's verdicts
            assert np.array_equal(after[0][m], oracle.verify_rec128(recs, mode=m))
        _audit_clean(e, node)
        e.committee_commit()
        node = Node(P)
        assert e.key_slots == 64
        _audit_clean(e, node)
        new_recs = _sign(oracle, all_seeds, all_pks, np.arange(32, 96), 644, corrupt=0.1)
        _verdicts_by_index(e, oracle, node, new_recs, np.arange(64, dtype=np.uint32))
    finally:
        e.close()


def test_window_changes_both_ways(oracle):
    """From no committee (key cache) to 10-bit windows, then 12, then 10 again: hs_window_bits follows and every verdict stays the
    oracle's."""
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 48, 650)
    recs = _sign(oracle, seeds, pks, np.arange(48).repeat(2), 651, corrupt=0.2)
    want = [oracle.verify_rec128(recs, mode=m) for m in (0, 1)]
    vidx = np.arange(48, dtype=np.uint32).repeat(2)
    e = Engine(0)
    try:
        for w in (10, 12, 10):
            valid, bits = e.committee_stage_register(pks, w)
            assert valid.all() and bits == w
            e.committee_commit()
            assert e.window_bits[0] == w and e.key_slots == 48
            for m in (0, 1):
                assert np.array_equal(e.verify_rec128(recs, mode=m), want[m])
            assert np.array_equal(e.verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(recs), dtype=np.uint32)), want[0])
            _audit_clean(e, Node(pks))
            assert e.self_test() == 0, e.last_error
    finally:
        e.close()


def _intact(e, oracle, node, recs, vidx):
    """The live committee still verifies as the oracle says and audits clean with its map."""
    _verdicts_by_index(e, oracle, node, recs, vidx)
    _audit_clean(e, node)


def test_errors_leave_the_live_committee_intact(oracle):
    import torch
    from hotstuff_b200 import Engine, EngineError
    seeds, pks = _keys(oracle, 40, 660)
    _, npks = _keys(oracle, 256, 661)
    e = Engine(0, key_window=12)
    lib = e.lib
    try:
        e.committee_register(pks)
        node = Node(pks)
        recs = _sign(oracle, seeds, pks, np.arange(40), 662, corrupt=0.2)
        vidx = np.arange(40, dtype=np.uint32)
        # a budget too small for any window
        e.set_table_budget(1 << 20)
        rc, bm, bits = _stage_register_raw(e, npks)
        assert rc == HS_ERR_NOMEM and (bm == 0xAAAAAAAA).all() and bits == -1
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        e.set_table_budget(0)
        _intact(e, oracle, node, recs, vidx)
        # argument errors write nothing
        for args in ((npks[:0], 0), (npks, 7), (npks, 18), (npks, 10)):  # N == 0, widths out of range, unlike the forced window
            rc, bm, bits = _stage_register_raw(e, *args)
            assert rc == HS_ERR_ARG and (bm == 0xAAAAAAAA).all() and bits == -1, args
        assert lib.hs_committee_stage_register(None, None, 0, 0, None, None) == HS_ERR_ARG
        # a second stage of either kind
        e.committee_stage_register(npks)
        for call in (lambda: e.committee_stage_register(npks), lambda: e.committee_stage(npks[:1])):
            with pytest.raises(EngineError):
                call()
        e.committee_discard()
        e.committee_stage(npks[:1])
        assert _stage_register_raw(e, npks)[0] == HS_ERR_ARG
        e.committee_discard()
        # a registration or an update during the stage discards it
        e.committee_stage_register(npks)
        e.committee_register(pks)
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        _intact(e, oracle, node, recs, vidx)
        e.committee_stage_register(npks)
        idx = e.committee_update(npks[:1], [39])
        node.update(npks[:1], idx, [39])
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        _audit_clean(e, node)
        e.committee_register(pks)
        node = Node(pks)
        # discard frees the staged store
        torch.cuda.mem_get_info(0)  # the first call sets torch's own context up
        free0 = torch.cuda.mem_get_info(0)[0]
        e.committee_stage_register(npks)
        staged = free0 - torch.cuda.mem_get_info(0)[0]
        assert staged > 256 * 2 ** 20, staged  # 272 slots of 12-bit tables
        e.committee_discard()
        assert torch.cuda.mem_get_info(0)[0] - (free0 - staged) > staged * 0.9  # given back
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        _intact(e, oracle, node, recs, vidx)
        # an audit, a repair or a mend leaves it pending
        e.committee_stage_register(npks)
        _audit_clean(e, node)
        assert e.table_repair(pks)[1] == 0
        assert e.table_mend(pks)[1] == 0
        e.committee_commit()
        assert e.key_slots == 256
        _audit_clean(e, Node(npks))
    finally:
        e.close()


def test_a_corrupt_staged_table_fails_its_proof(oracle, hooklib):
    hooklib.hs_test_poke_staged.restype = ctypes.c_int
    hooklib.hs_test_poke_staged.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint8]
    seeds, pks = _keys(oracle, 40, 670)
    _, npks = _keys(oracle, 48, 671)
    h = _engine(hooklib, key_window=12)
    try:
        h.committee_register(pks)
        node = Node(pks)
        recs = _sign(oracle, seeds, pks, np.arange(40), 672, corrupt=0.2)
        vidx = np.arange(40, dtype=np.uint32)
        l0 = h.kernel_launches
        assert hooklib.hs_test_poke_staged(h.h, POKE_TABLE, 7, _entry_off(12, 1, 3), 0x10) == 0
        rc, bm, bits = _stage_register_raw(h, npks)
        assert rc == HS_ERR_SELFTEST and "slot 7: comb table" in h.last_error and (bm == 0xAAAAAAAA).all() and bits == -1, h.last_error
        assert h.kernel_launches - l0 == 3  # one build, the slot checks, the tables
        assert hooklib.hs_committee_commit(h.h) == HS_ERR_ARG
        _intact(h, oracle, node, recs, vidx)
        # the next stage is clean, and commits
        valid, bits = h.committee_stage_register(npks)
        assert valid.all() and bits == 12
        h.committee_commit()
        _audit_clean(h, Node(npks))
    finally:
        h.close()


def test_votes_across_the_stage_and_the_commit(oracle):
    """A 667-vote queue burst from 16 threads, with the signature cache on and shared, while a 512-key registration is staged and
    committed: every vote gets the oracle's verdict, and a record cached before the commit still hits after it."""
    from hotstuff_b200 import Engine
    e = Engine(0, key_window=12)
    try:
        rng = np.random.default_rng(680)
        seeds = np.frombuffer(rng.bytes(32 * 1024), np.uint8).reshape(-1, 32).copy()
        allpks = e.keygen_batch(seeds)
        pks, P = allpks[:512], allpks[256:768]  # the staged committee keeps half the validators
        e.committee_register(pks)
        ki = rng.choice(512, 667, replace=True)
        dig = np.frombuffer(rng.bytes(32), np.uint8)
        sig = e.sign_digests(seeds[:512], pks, np.tile(dig, (667, 1)), key_idx=ki.astype(np.uint32))
        recs = np.concatenate([sig, pks[ki], np.tile(dig, (667, 1))], axis=1)
        for i in rng.choice(667, 40, replace=False):
            recs[i, rng.integers(0, 64)] ^= 1
        want = oracle.verify_rec128(recs)
        got = np.zeros(667, bool)
        with e.queue() as q:
            q.sig_cache(4096)
            q.sig_share(True)
            first = q.wait(q.submit(recs[:1]))[0]
            assert first == want[0]
            res = {}

            def change():
                res["valid"] = e.committee_stage_register(P, 12)[0]
                e.committee_commit()

            th = threading.Thread(target=change)
            th.start()

            def worker(t):
                for i in range(t, 667, 16):
                    got[i] = q.wait(q.submit(recs[i:i + 1]))[0]

            ws = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
            for w in ws:
                w.start()
            for w in ws:
                w.join()
            th.join()
            assert np.array_equal(got, want)
            hits = q.sig_stats()["hits"]
            assert q.wait(q.submit(recs[:1]))[0] == want[0]
            if want[0]:
                assert q.sig_stats()["hits"] > hits  # cached before the commit, a hit after it
        assert res["valid"].all() and e.key_slots == 512
        _audit_clean(e, Node(P))
    finally:
        e.close()


def test_multi_engine_discards_on_every_member_when_one_fails(oracle):
    from hotstuff_b200 import EngineError, MultiEngine
    seeds, pks = _keys(oracle, 48, 690)
    nseeds, npks = _keys(oracle, 64, 691)
    m = MultiEngine([0, 0], key_window=12)
    try:
        m.register_committee(pks)
        node = Node(pks)
        recs = _sign(oracle, seeds, pks, np.arange(48), 692, corrupt=0.2)
        vidx = np.arange(48, dtype=np.uint32)
        m.member(1).set_table_budget(1 << 20)
        with pytest.raises(EngineError):
            m.stage_register_committee(npks)
        for i in range(len(m)):
            assert m.lib.hs_committee_commit(m.member(i).h) == HS_ERR_ARG  # nothing stays staged
            _intact(m.member(i), oracle, node, recs, vidx)
        m.member(1).set_table_budget(0)
        valid, bits = m.stage_register_committee(npks)
        assert valid.all() and bits == 12
        m.commit_committee()
        node = Node(npks)
        new_recs = _sign(oracle, nseeds, npks, np.arange(64), 693, corrupt=0.2)
        for i in range(len(m)):
            _intact(m.member(i), oracle, node, new_recs, np.arange(64, dtype=np.uint32))
    finally:
        m.close()
