"""hs_table_mend: corrupt comb-table entries mended in place, with no drain and no slot out of service.

GPU, on the engine built with the corruption hook (hs_test_poke, -DHS_TEST_HOOKS, as tests/test_table_repair.py builds it): poked
entries of the base-point table and of per-key tables at every forced key window are mended and proven by a clean audit, the slots stay
in service throughout and verify as the oracle does, votes keep completing while a 24-bit base window is mended, what the mend cannot
fix is left to hs_table_repair, the caches are emptied only when an entry was rewritten, and the scrub mends when told to."""
import ctypes
import threading
import time

import numpy as np
import pytest

from test_table_repair import (HS_AUDIT_BASE, HS_AUDIT_FLAG, HS_AUDIT_KEY, HS_AUDIT_TABLE, POKE_BASE, POKE_FLAG, POKE_KEY, POKE_TABLE,
                               _adversarial, _all_paths_match, _committee, _engine, _entry_off, _expect_clean, _keys, _last, _live_bits,
                               _poke, _windows, big, hooklib)  # noqa: F401  (fixtures)

HS_AUDIT_LOOKUP = 4
ZERO_STATS = {"windows_recomputed": 0, "entries_rewritten": 0, "windows_left": 0, "slots_left": 0, "cache_flushes": 0}


def _stats_delta(eng, before):
    after = eng.mend_stats()
    return {k: after[k] - before[k] for k in after}


@pytest.mark.gpu
def test_a_clean_context_is_one_audit_and_writes_nothing(big):
    eng, seeds, pks = big
    recs, _ = _adversarial(eng, seeds, pks, range(64), 256, 1)
    q = eng.queue()
    try:
        q.sig_cache(1 << 14)
        q.cert_cache(1 << 20)
        q.wait(q.submit_group(recs))
        launches, before, caches = eng.kernel_launches, eng.mend_stats(), (q.sig_stats(), q.cert_stats())
        found, left, bits = eng.table_mend(pks)
        assert (found, left) == (0, 0) and not bits.any()
        assert eng.kernel_launches - launches == 3  # one audit: k_slot_audit and k_table_audit over the key and base tables
        assert _stats_delta(eng, before) == dict(ZERO_STATS, calls=1)
        assert (q.sig_stats(), q.cert_stats()) == caches
    finally:
        q.close()


@pytest.mark.gpu
def test_base_entries(hooklib, oracle, golden):
    eng = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _committee(eng, golden, 64, 110)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        wb = eng.window_bits[1]
        stride = (1 << (wb - 1)) + 1
        last_win, last_m = _last(wb)
        mid = _windows(wb) // 2
        for index, byte in ((1, 3), (mid * stride + 1000, 50), (last_win * stride + last_m, 90)):
            _poke(eng, POKE_BASE, index, byte)
        assert eng.table_audit()[0] == HS_AUDIT_BASE
        before = eng.mend_stats()
        found, left, bits = eng.table_mend(pks)
        assert (found, left) == (HS_AUDIT_BASE, 0) and not bits.any(), eng.last_error
        d = _stats_delta(eng, before)
        assert d["entries_rewritten"] == 3 and d["windows_left"] == 0 and d["slots_left"] == 0 and d["cache_flushes"] == 1
        assert 3 <= d["windows_recomputed"] <= 5  # the anchor's window 0, the middle window, the last; a link may add its neighbour
        _expect_clean(eng, pks)
        assert eng.self_test() == 0, eng.last_error
        recs, ki = _adversarial(eng, seeds, pks, range(64), 512, 111)
        _all_paths_match(eng, oracle, recs, ki)
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key_bits", list(range(8, 18)))
def test_key_entries_stay_in_service(hooklib, oracle, golden, key_bits):
    # A forced window does not shrink to the free memory: a small committee and a 16-bit base table, as in test_table_repair.
    eng = _engine(hooklib, base_window=16, key_window=key_bits)
    try:
        seeds, pks = _committee(eng, golden, 24, 120 + key_bits)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        W = eng.window_bits[0]
        assert W == key_bits
        H, top = 1 << (W - 1), _windows(W) - 1
        # the anchor (entry 1 of window 0), a link entry (2^(w-1) of a middle window), entry 1 of a later window, the last entry
        spots = {3: (0, 1, 5), 7: (top // 2, H, 40), 11: (top, 1, 70), 15: (top, H, 20), 19: (1, 3, 33)}
        for s, (win, m, byte) in spots.items():
            _poke(eng, POKE_TABLE, s, _entry_off(W, win, m, byte))
        slots = sorted(spots)
        votes, ki = _adversarial(eng, seeds, pks, slots, 300, 121 + key_bits)
        q = eng.queue()
        try:
            st0, g0 = q.stats(), q.generic_stats()
            before = eng.mend_stats()
            found, left, bits = eng.table_mend(pks)
            assert (found, left) == (HS_AUDIT_TABLE, 0), eng.last_error
            assert sorted(np.nonzero(bits)[0]) == slots
            d = _stats_delta(eng, before)
            assert d["entries_rewritten"] == len(spots) and d["slots_left"] == 0
            # the slots never left service: their votes take neither the slow path nor the generic lane
            want = oracle.verify_rec128(votes)
            got = [q.wait(q.submit(votes[i:i + 1]))[0] for i in range(64)]
            assert np.array_equal(np.array(got, bool), want[:64])
            st1, g1 = q.stats(), q.generic_stats()
            assert (st1["slow_requests"], st1["slow_records"]) == (st0["slow_requests"], st0["slow_records"])
            assert g1 == g0
        finally:
            q.close()
        _expect_clean(eng, pks)
        _all_paths_match(eng, oracle, votes, ki)
    finally:
        eng.close()


def _vote_stream(q, vote, stop, out):
    """One vote at a time until `stop` is set: (verdict, latency) each."""
    while not stop.is_set():
        t = time.perf_counter()
        v = q.wait(q.submit(vote))[0]
        out.append((bool(v), time.perf_counter() - t))


@pytest.mark.gpu
def test_votes_complete_while_a_24_bit_base_window_is_mended(big, oracle):
    eng, seeds, pks = big
    wb = eng.window_bits[1]
    if wb != 24:
        pytest.skip("the base-point table is %d bits wide on this device" % wb)
    stride = (1 << 23) + 1
    vote, _ = _adversarial(eng, seeds, pks, [9], 1, 130)
    want = bool(oracle.verify_rec128(vote)[0])
    # a high entry of window 5: a vote gathers it with probability about 2^-23, so verdicts are exact before and after
    _poke(eng, POKE_BASE, 5 * stride + (1 << 23) - 3, 11)
    q = eng.queue()
    try:
        q.wait(q.submit(vote))
        stop, lat, res = threading.Event(), [], {}
        th = threading.Thread(target=_vote_stream, args=(q, vote, stop, lat))
        t0 = time.perf_counter()
        mend = threading.Thread(target=lambda: res.setdefault("r", eng.table_mend(pks)))
        mend.start()
        th.start()
        mend.join()
        t_mend = time.perf_counter() - t0
        n_during = len(lat)
        stop.set()
        th.join()
    finally:
        q.close()
    found, left, _ = res["r"]
    assert (found, left) == (HS_AUDIT_BASE, 0), eng.last_error
    assert all(v == want for v, _ in lat)
    # votes went on throughout: many completed during the mend, none waited anywhere near its length (a repair holds them all)
    assert n_during >= 10, (n_during, t_mend)
    assert max(t for _, t in lat[:n_during]) < t_mend / 2, (max(t for _, t in lat), t_mend)
    _expect_clean(eng, pks)


@pytest.mark.gpu
def test_key_and_flag_findings_are_left_to_the_repair(hooklib, oracle, golden):
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 200, 140)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        W = eng.window_bits[0]
        _poke(eng, POKE_KEY, 20, 4)
        _poke(eng, POKE_FLAG, 9, 0, 0x01)
        _poke(eng, POKE_TABLE, 30, _entry_off(W, 2, 9))
        before = eng.mend_stats()
        found, left, bits = eng.table_mend(pks)
        # changed key bytes also miss the hash table (LOOKUP) and no longer match their table's anchor (TABLE): slot 20 is left whole
        every = HS_AUDIT_KEY | HS_AUDIT_FLAG | HS_AUDIT_LOOKUP | HS_AUDIT_TABLE
        assert (found, left) == (every, every), eng.last_error
        assert "hs_table_repair" in eng.last_error
        assert sorted(np.nonzero(bits)[0]) == [9, 20, 30]
        d = _stats_delta(eng, before)
        assert d["slots_left"] == 2 and d["entries_rewritten"] == 1
        failed, abits = eng.table_audit(pks)
        assert sorted(np.nonzero(abits)[0]) == [9, 20] and abits[20] & HS_AUDIT_TABLE  # slot 30 mended, the rest untouched
        found, failed, _ = eng.table_repair(pks)
        assert failed == 0 and found == every, eng.last_error
        _expect_clean(eng, pks)
        recs, ki = _adversarial(eng, seeds, pks, [9, 20, 30], 300, 141)
        _all_paths_match(eng, oracle, recs, ki)
    finally:
        eng.close()


@pytest.mark.gpu
def test_an_anchor_is_mended_only_with_a_map(hooklib, oracle, golden):
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 100, 150)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        W = eng.window_bits[0]
        _poke(eng, POKE_TABLE, 5, _entry_off(W, 0, 1, 3))
        found, left, bits = eng.table_mend()
        assert (found, left) == (HS_AUDIT_TABLE, HS_AUDIT_TABLE) and list(np.nonzero(bits)[0]) == [5]
        assert eng.table_audit()[0] == HS_AUDIT_TABLE  # untouched
        found, left, _ = eng.table_mend(pks)
        assert (found, left) == (HS_AUDIT_TABLE, 0), eng.last_error
        _expect_clean(eng, pks)
        recs, ki = _adversarial(eng, seeds, pks, [5], 200, 151)
        _all_paths_match(eng, oracle, recs, ki)
    finally:
        eng.close()


@pytest.mark.gpu
def test_caches_are_emptied_only_when_an_entry_was_rewritten(big, oracle):
    eng, seeds, pks = big
    W = eng.window_bits[0]
    votes, _ = _adversarial(eng, seeds, pks, list(range(300)), 300, 160)
    q = eng.queue()
    try:
        q.sig_cache(1 << 14)
        q.cert_cache(1 << 20)
        dig = np.frombuffer(np.random.default_rng(161).bytes(32), np.uint8)
        qc_ki = np.arange(200, 300, dtype=np.uint32)
        qc = np.zeros((100, 128), np.uint8)
        qc[:, :64] = eng.sign_digests(seeds, pks, np.tile(dig, (100, 1)), key_idx=qc_ki)
        qc[:, 64:96], qc[:, 96:] = pks[qc_ki], dig
        assert q.wait(q.submit_group(qc, modes=np.ones(100, np.uint8))).all()
        for i in range(0, 300, 30):
            q.wait(q.submit(votes[i:i + 30]))
        held = (q.sig_stats()["entries_held"], q.cert_stats()["bytes_held"])
        assert held[0] > 0 and held[1] > 0
        # a finding the mend leaves (a flag byte) rewrites nothing: the caches stay
        _poke(eng, POKE_FLAG, 3000, 0, 0x02)
        assert eng.table_mend(pks)[1] == HS_AUDIT_FLAG
        assert (q.sig_stats()["entries_held"], q.cert_stats()["bytes_held"]) == held
        assert eng.table_repair(pks)[1] == 0, eng.last_error
        assert q.wait(q.submit_group(qc, modes=np.ones(100, np.uint8))).all()
        assert q.sig_stats()["entries_held"] > 0
        _poke(eng, POKE_TABLE, 7, _entry_off(W, 2, 9))
        found, left, _ = eng.table_mend(pks)
        assert (found, left) == (HS_AUDIT_TABLE, 0), eng.last_error
        assert q.sig_stats()["entries_held"] == 0 and q.cert_stats()["bytes_held"] == 0
        assert q.wait(q.submit_group(qc, modes=np.ones(100, np.uint8))).all()
    finally:
        q.close()


@pytest.mark.gpu
def test_the_scrub_mends_when_told_to(hooklib, golden):
    eng = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _committee(eng, golden, 64, 170)
        eng.committee_register(pks)
        W, wb = eng.window_bits
        calls = []
        eng.scrub_mend(True)
        _poke(eng, POKE_BASE, 3 * ((1 << (wb - 1)) + 1) + 77, 8)
        _poke(eng, POKE_TABLE, 40, _entry_off(W, 1, 6))
        before = eng.mend_stats()
        eng.scrub_start(pks, period_us=2000, slots_per_tick=64, base_entries_per_tick=1 << 22,
                        callback=lambda found, failed, first: calls.append((found, failed, first)))
        t = time.time()
        while not calls and time.time() - t < 20:
            time.sleep(0.01)
        eng.scrub_stop()
        assert calls and calls[0] == (HS_AUDIT_BASE | HS_AUDIT_TABLE, 0, 40), calls
        d = _stats_delta(eng, before)
        assert d["calls"] >= 1 and d["entries_rewritten"] == 2 and d["slots_left"] == 0
        st = eng.scrub_stats()
        assert st["slots_repaired"] == 0 and st["failed_repairs"] == 0 and st["findings"] >= 2
        _expect_clean(eng, pks)
        # a finding the mend cannot fix is repaired, as without hs_scrub_mend
        calls.clear()
        _poke(eng, POKE_FLAG, 12, 0, 0x01)
        eng.scrub_start(pks, period_us=2000, slots_per_tick=64, base_entries_per_tick=1 << 22,
                        callback=lambda found, failed, first: calls.append((found, failed, first)))
        t = time.time()
        while not calls and time.time() - t < 20:
            time.sleep(0.01)
        eng.scrub_stop()
        assert calls and calls[0] == (HS_AUDIT_FLAG, 0, 12), calls
        assert eng.scrub_stats()["slots_repaired"] == 1
        _expect_clean(eng, pks)
    finally:
        eng.close()


@pytest.mark.gpu
def test_an_update_racing_a_mend_never_leaves_a_wrong_table(hooklib, golden):
    from hotstuff_b200 import EngineError
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 1000, 180)
        _, extra = _keys(eng, 8, 181)
        eng.committee_register(pks)
        W = eng.window_bits[0]
        node = [bytes(k) for k in pks]
        for it in range(4):
            for s in range(100 + 10 * it, 108 + 10 * it):
                _poke(eng, POKE_TABLE, s, _entry_off(W, 1, 2 + s))
            res = {}

            def mend():
                try:
                    res["r"] = eng.table_mend()
                except EngineError as e:
                    res["e"] = str(e)

            th = threading.Thread(target=mend)
            th.start()
            time.sleep(0.002 * it)
            idx = eng.committee_update(extra[it:it + 1], [it])
            th.join()
            node[it] = None
            for k, i in zip(extra[it:it + 1], idx):
                while i >= len(node):
                    node.append(None)
                node[i] = bytes(k)
            if "r" in res:
                assert res["r"][1] == 0, eng.last_error
            else:
                assert "changed during the mend" in res["e"] or "changed during the audit" in res["e"], res["e"]
            exp = np.array([np.frombuffer(k, np.uint8) if k else np.zeros(32, np.uint8) for k in node], np.uint8)
            lv = _live_bits([k is not None for k in node])
            failed, bits = eng.table_audit(exp, lv)
            if failed:  # the mend lost the race before it stored anything: its findings are still there, and a mend now clears them
                assert failed == HS_AUDIT_TABLE, eng.last_error
                assert eng.table_mend(exp, lv)[1] == 0, eng.last_error
            _expect_clean(eng, exp, lv)
    finally:
        eng.close()


@pytest.mark.gpu
def test_argument_errors_write_nothing(hooklib):
    from hotstuff_b200 import EngineError
    eng = _engine(hooklib)
    try:
        _, pks = _keys(eng, 40, 190)
        eng.committee_register(pks)
        found, left = ctypes.c_uint32(77), ctypes.c_uint32(88)
        bits = np.full(40, 0xaa, np.uint8)
        lib = eng.lib
        before = eng.mend_stats()
        for n in (39, 41):
            assert lib.hs_table_mend(eng.h, None, None, n, bits.ctypes.data_as(ctypes.c_void_p), ctypes.byref(found), ctypes.byref(left)) == 2
        assert lib.hs_table_mend(eng.h, None, None, 40, None, None, ctypes.byref(left)) == 2
        assert lib.hs_table_mend(eng.h, None, None, 40, None, ctypes.byref(found), None) == 2
        assert lib.hs_table_mend(None, None, None, 0, None, ctypes.byref(found), ctypes.byref(left)) == 2
        assert lib.hs_table_mend_stats(eng.h, None) == 2 and lib.hs_scrub_mend(None, 1) == 2
        assert (found.value, left.value) == (77, 88) and (bits == 0xaa).all()
        with pytest.raises(EngineError):
            eng.table_mend(pks[:-1])
        assert eng.mend_stats() == before
        _expect_clean(eng, pks)
    finally:
        eng.close()
