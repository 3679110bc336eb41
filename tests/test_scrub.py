"""hs_scrub_*: the engine-owned scrub of the live key tables, on the GPU.

Real corrupt bytes (hs_test_poke, on a build with -DHS_TEST_HOOKS, as in test_table_repair.py) in a comb table, a flag byte, key bytes
(which also break the slot's hash lookup) and the base-point table are each found and repaired within one pass, reach the callback once
and are counted; verdicts afterwards are the oracle's.  A clean committee gives no finding over several passes, with the pass count the
slice sizes predict.  A committee change pauses the scrub until the new map, a stage and commit under a running scrub equal two updates,
a verify-queue burst beside the scrub gets the oracle's verdicts, and stop / destroy leave no thread.  Every wait below polls the
counters until they advance (with a bound that only guards against a hang); nothing passes or fails on a time."""
import os
import threading
import time

import numpy as np
import pytest

from test_committee_stage import Node, _audit_clean, _keys, _sign
from test_table_repair import (HS_AUDIT_BASE, HS_AUDIT_FLAG, HS_AUDIT_KEY, HS_AUDIT_LOOKUP, HS_AUDIT_TABLE, POKE_BASE, POKE_FLAG,
                               POKE_KEY, POKE_TABLE, _adversarial, _all_paths_match, _committee, _engine, _entry_off, _golden_recs,
                               _poke, _windows, hooklib)  # noqa: F401  (hooklib: the fixture)

pytestmark = pytest.mark.gpu
NONE = (1 << 64) - 1  # first_slot when only the base-point table or a stray hash entry was found


class Findings:
    """The scrub's callback: every call, in order, taken on the scrub's thread."""

    def __init__(self):
        self.calls, self.lock = [], threading.Lock()

    def __call__(self, found, failed, first_slot):
        with self.lock:
            self.calls.append((found, failed, first_slot))


def _wait(eng, what, pred, bound_s=300):
    """Polls scrub_stats() until pred(stats); the bound only stops a hung scrub from hanging the suite."""
    end = time.monotonic() + bound_s
    while True:
        st = eng.scrub_stats()
        if pred(st):
            return st
        assert time.monotonic() < end, "%s: the scrub did not get there: %s (%s)" % (what, st, eng.last_error)
        time.sleep(0.005)


def _passes(eng, k, base=0):
    return _wait(eng, "%d passes" % k, lambda st: st["passes"] >= base + k)


def _base_entries(eng):
    return _windows(eng.window_bits[1]) * ((1 << (eng.window_bits[1] - 1)) + 1)


def _scrub_threads():
    """Threads of this process named as the scrub names its thread."""
    n = 0
    for t in os.listdir("/proc/self/task"):
        try:
            with open("/proc/self/task/%s/comm" % t) as f:
                n += f.read().strip() == "hs_scrub"
        except OSError:  # the thread ended meanwhile
            pass
    return n


@pytest.fixture
def big(hooklib, golden):
    """A 4 096-key committee at the window the budget picks, with the default 24-bit base-point table (8.9 GB)."""
    eng = _engine(hooklib)
    seeds, pks = _committee(eng, golden, 4096, 91)
    assert eng.committee_register(pks).all()
    eng._pks_for_test = pks
    yield eng, seeds, pks
    eng.close()


def test_clean_committee_passes_as_predicted_beside_a_queue_burst(big, oracle):
    """No finding over several passes; a pass is max(ceil(4096 / slots), ceil(E / base entries)) = 4 ticks.  The base slices are not
    window-aligned, so every window boundary but one is crossed inside a slice.  A 667-vote burst through the verify queue while the
    scrub runs gets the oracle's verdicts."""
    eng, seeds, pks = big
    E = _base_entries(eng)
    per_tick = -(-E // 4)
    fired = Findings()
    eng.scrub_start(pks, None, period_us=500, slots_per_tick=1024, base_entries_per_tick=per_tick, callback=fired)
    try:
        recs, _ = _adversarial(eng, seeds, pks, range(4096), 667, 92)
        want = oracle.verify_rec128(recs, mode=0)
        q = eng.queue()
        try:
            tickets = [q.submit(recs[i:i + 1]) for i in range(len(recs))]
            got = np.array([q.wait(t)[0] for t in tickets], bool)
            assert np.array_equal(got, want)
        finally:
            q.close()
        _passes(eng, 3)
    finally:
        eng.scrub_stop()
    st = eng.scrub_stats()
    assert fired.calls == [] and st["findings"] == st["slots_repaired"] == st["failed_repairs"] == st["ticks_paused"] == 0, st
    assert st["passes"] == st["ticks"] // 4, st
    assert st["slots_audited"] == 1024 * st["ticks"], st
    done = st["ticks"] % 4
    assert st["base_entries_audited"] == st["passes"] * E + done * per_tick, st
    assert eng.table_audit(pks)[0] == 0, eng.last_error


def test_each_corruption_is_found_and_repaired_within_one_pass(big, oracle, golden):
    """A comb-table entry (slot 3000, a middle window), a flag byte (slot 9), a key byte (slot 20: KEY against the map, and its lookup
    and table anchor break with it) and a base-point entry (the last entry of a middle window, whose link to the next window breaks too),
    poked before the scrub starts: found and repaired in the first pass, counted once each, every callback reporting a clean repair."""
    eng, seeds, pks = big
    W, Wb = eng.window_bits
    mid = _windows(W) // 2
    _poke(eng, POKE_TABLE, 3000, _entry_off(W, mid, 7))
    _poke(eng, POKE_FLAG, 9, 0, 0x01)
    _poke(eng, POKE_KEY, 20, 4)
    bw = _windows(Wb) // 2
    _poke(eng, POKE_BASE, bw * ((1 << (Wb - 1)) + 1) + (1 << (Wb - 1)), 9)
    failed, bits = eng.table_audit(pks)
    assert failed == HS_AUDIT_KEY | HS_AUDIT_FLAG | HS_AUDIT_LOOKUP | HS_AUDIT_TABLE | HS_AUDIT_BASE
    assert sorted(np.nonzero(bits)[0]) == [9, 20, 3000]
    fired = Findings()
    E = _base_entries(eng)
    eng.scrub_start(pks, None, period_us=500, slots_per_tick=512, base_entries_per_tick=-(-E // 8), callback=fired)
    try:
        _passes(eng, 1)
        after_one = list(fired.calls)
        _passes(eng, 3)
    finally:
        eng.scrub_stop()
    st = eng.scrub_stats()
    assert fired.calls == after_one, "a finding reached the callback after the first pass: %s" % fired.calls
    assert all(failed == 0 for _, failed, _ in fired.calls), fired.calls
    found = 0
    for f, _, _ in fired.calls:
        found |= f
    assert found == HS_AUDIT_KEY | HS_AUDIT_FLAG | HS_AUDIT_LOOKUP | HS_AUDIT_TABLE | HS_AUDIT_BASE, fired.calls
    assert fired.calls[0][2] == 9  # the slot checks run over every slot in the first tick
    assert st["findings"] == 4 and st["slots_repaired"] == 3 and st["failed_repairs"] == 0, st
    failed, bits = eng.table_audit(pks)
    assert failed == 0 and not bits.any(), eng.last_error
    recs, ki = _adversarial(eng, seeds, pks, [9, 20, 3000, 3001], 768, 93)
    _all_paths_match(eng, oracle, recs, ki)
    g = _golden_recs(golden)
    assert np.array_equal(eng.verify_rec128(g), oracle.verify_rec128(g))


def _key_poke(oracle, key, decompresses):
    """(byte, mask) of a one-bit change to `key` whose result does, or does not, decompress."""
    for byte in range(31):
        for bit in range(8):
            k = bytearray(key.tobytes())
            k[byte] ^= 1 << bit
            if oracle.decompress_ok(bytes(k)) == decompresses:
                return byte, 1 << bit
    raise AssertionError("no such change")


def test_key_bytes_without_a_map(hooklib, oracle, golden):
    """Against the engine's own mirror the slot checks cannot tell changed key bytes wrong: they see LOOKUP, and FLAG when the new bytes
    do not decompress.  The tick that flags a slot also audits its table, outside its slice, and the anchor (TABLE) is what makes the
    repair rebuild a slot whose new bytes decompress.  One bit in each of two slots, far ahead of the cursor: one callback, both
    repaired from the mirror."""
    eng = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _committee(eng, golden, 200, 94)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        _poke(eng, POKE_KEY, 150, *_key_poke(oracle, pks[150], True))
        _poke(eng, POKE_KEY, 170, *_key_poke(oracle, pks[170], False))
        fired = Findings()
        # a slot a tick: the first tick's slice is slot 0, and its slot checks flag 150 and 170
        eng.scrub_start(None, None, period_us=500, slots_per_tick=1, base_entries_per_tick=1 << 20, callback=fired)
        try:
            _passes(eng, 2)
        finally:
            eng.scrub_stop()
        st = eng.scrub_stats()
        assert fired.calls == [(HS_AUDIT_FLAG | HS_AUDIT_LOOKUP | HS_AUDIT_TABLE, 0, 150)], fired.calls
        assert st["findings"] == 2 and st["slots_repaired"] == 2 and st["failed_repairs"] == 0, st
        assert eng.table_audit(pks)[0] == 0, eng.last_error
        _all_paths_match(eng, oracle, *_adversarial(eng, seeds, pks, [150, 151, 170], 256, 95))
    finally:
        eng.close()


def test_base_entries_across_a_window_boundary(hooklib):
    """Slices of a prime number of entries cross window boundaries at every offset.  Entry 1 of a window (its link to the window
    before) and the last entry of the window before it, poked apart: the scrub finds the base-point table as the full audit does, once,
    and leaves it clean."""
    eng = _engine(hooklib, base_window=16)
    try:
        stride = (1 << 15) + 1
        for e in (5 * stride + 1, 9 * stride - 1):
            _poke(eng, POKE_BASE, e, 40)
            assert eng.table_audit()[0] == HS_AUDIT_BASE
            fired = Findings()
            eng.scrub_start(None, None, period_us=300, slots_per_tick=1, base_entries_per_tick=10007, callback=fired)
            try:
                _passes(eng, 2)
            finally:
                eng.scrub_stop()
            assert fired.calls == [(HS_AUDIT_BASE, 0, NONE)], fired.calls
            st = eng.scrub_stats()
            assert st["findings"] == 1 and st["failed_repairs"] == 0 and st["slots_repaired"] == 0, st
            assert eng.table_audit()[0] == 0, eng.last_error
    finally:
        eng.close()


def test_a_committee_change_pauses_until_the_new_map(oracle):
    """After an update the scrub pauses, finding nothing, until scrub_set_map gives the new map; then it resumes cleanly."""
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 120, 96)
    _, npks = _keys(oracle, 3, 97)
    eng = Engine(0, base_window=16, key_window=10)
    try:
        eng.committee_register(pks)
        node = Node(pks)
        fired = Findings()
        exp, lv = node.expect()
        eng.scrub_start(exp, lv, period_us=300, slots_per_tick=40, base_entries_per_tick=1 << 17, callback=fired)
        try:
            _passes(eng, 1)
            idx = eng.committee_update(npks, [4, 77])
            node.update(npks, idx, [4, 77])
            paused = eng.scrub_stats()["ticks_paused"]
            _wait(eng, "pauses", lambda st: st["ticks_paused"] >= paused + 5)
            exp, lv = node.expect()
            eng.scrub_set_map(exp, lv)
            base = eng.scrub_stats()
            _passes(eng, 2, base["passes"])
        finally:
            eng.scrub_stop()
        st = eng.scrub_stats()
        assert fired.calls == [] and st["findings"] == 0, (fired.calls, st)
        assert st["ticks"] > base["ticks"]
        _audit_clean(eng, node)
    finally:
        eng.close()


def test_stage_and_commit_under_a_scrub_equal_two_updates(oracle):
    """stage(A, R) + commit on a context whose scrub runs, update(A) + update(remove=R) on another: the same indices and slots, clean
    audits against the same map, the same verdicts, and the scrub resumes on the new map without a finding."""
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 150, 98)
    nseeds, npks = _keys(oracle, 5, 99)
    e1, e2 = Engine(0, base_window=16, key_window=10), Engine(0, base_window=16, key_window=10)
    try:
        node = Node(pks)
        for e in (e1, e2):
            e.committee_register(pks)
        fired = Findings()
        e1.scrub_start(pks, None, period_us=300, slots_per_tick=32, base_entries_per_tick=1 << 17, callback=fired)
        try:
            _passes(e1, 1)
            R = np.array([3, 60, 61], np.uint32)
            idx1 = e1.committee_stage(npks, R)
            e1.committee_commit()
            idx2 = e2.committee_update(npks)
            e2.committee_update(remove=R)
            assert np.array_equal(idx1, idx2)
            node.apply(npks, idx1, R)
            exp, lv = node.expect()
            e1.scrub_set_map(exp, lv)
            _passes(e1, 2, e1.scrub_stats()["passes"])
        finally:
            e1.scrub_stop()
        assert fired.calls == [] and e1.scrub_stats()["findings"] == 0
        assert e1.key_slots == e2.key_slots
        _audit_clean(e1, node)
        _audit_clean(e2, node)
        all_seeds, all_pks = np.concatenate([seeds, nseeds]), np.concatenate([pks, npks])
        ki = np.array(list(range(150, 155)) * 8 + [3, 60, 61, 0, 1, 2] * 6, np.int64)
        recs = _sign(oracle, all_seeds, all_pks, ki, 100)
        want = oracle.verify_rec128(recs)
        for e in (e1, e2):
            assert np.array_equal(e.verify_rec128(recs), want)
    finally:
        e1.close()
        e2.close()


def test_lifecycle(oracle):
    """One scrub per context; stop joins its thread and is idempotent; audits and repairs beside it return what they return without
    it; destroying a context with a running scrub leaves no thread."""
    from hotstuff_b200 import Engine
    from hotstuff_b200.engine import EngineError
    _, pks = _keys(oracle, 40, 101)
    eng = Engine(0, base_window=16, key_window=8)
    try:
        eng.committee_register(pks)
        assert _scrub_threads() == 0
        eng.scrub_start(pks, None, period_us=200, slots_per_tick=8, base_entries_per_tick=1 << 16)
        _passes(eng, 1)
        assert _scrub_threads() == 1
        with pytest.raises(EngineError):
            eng.scrub_start(pks, None, period_us=200, slots_per_tick=8, base_entries_per_tick=1 << 16)
        with pytest.raises(EngineError):
            eng.scrub_set_map(pks[:10])  # not the slots in use
        _passes(eng, 1)
        assert eng.table_audit(pks)[0] == 0
        assert eng.table_repair(pks)[:2] == (0, 0)
        eng.scrub_stop()
        eng.scrub_stop()
        assert _scrub_threads() == 0
        st = eng.scrub_stats()
        assert st["passes"] >= 1 and st["findings"] == 0, st
        eng.scrub_start(None, None, period_us=200, slots_per_tick=8, base_entries_per_tick=1 << 16)
        assert eng.scrub_stats()["passes"] == 0  # a new scrub counts from zero
        _passes(eng, 1)
    finally:
        eng.close()  # hs_ctx_destroy with the scrub running
    assert _scrub_threads() == 0
