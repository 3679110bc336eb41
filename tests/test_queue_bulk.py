"""Large certificates on the verify queue's bulk kernel (k_verify_bulk): a device request of HS_QUEUE_BULK_MIN records or more gets a
launch of its own, a thread per signature, on the queue's second stream.  Every verdict must equal the oracle and hs_verify_rec128 on
that record in its mode, and the queue's counters (hs_queue_stats) must show each request on the kernel the threshold names."""
import os
import re
import threading

import numpy as np
import pytest

from oracle_api import make_workload, to_rec128
from test_queue_groups import _check, _clear, _committee, _expect, _run_group_threads, _submit, _threads, block_modes, pool  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BULK_MIN = int(re.search(r"#define HS_QUEUE_BULK_MIN (\d+)", open(os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")).read()).group(1))


def _delta(after, before):
    return {k: after[k] - before[k] for k in after}


def _lone(engine, q, pool, idx, modes):
    """One group with nothing else pending: its verdicts, its launches and the change of the queue's counters."""
    s0, l0 = q.stats(), engine.kernel_launches
    bits = q.wait(_submit(q, pool[0][idx], modes))
    assert (bits == _expect(pool, idx, modes)).all(), np.flatnonzero(bits != _expect(pool, idx, modes))[:8]
    return engine.kernel_launches - l0, _delta(q.stats(), s0)


def _routed(d, n, bulk):
    if bulk:
        return d == dict(small_launches=0, small_records=0, bulk_launches=1, bulk_records=n, slow_requests=0, slow_records=0)
    return d == dict(small_launches=1, small_records=n, bulk_launches=0, bulk_records=0, slow_requests=0, slow_records=0)


def test_threshold_is_above_the_small_request_limit():
    assert BULK_MIN > 64


@pytest.mark.parametrize("n,ring", [(BULK_MIN - 1, 4096), (BULK_MIN, 4096), (BULK_MIN + 1, 4096), (668, 4096), (6668, 16384)])
def test_lone_group_parity_kernel_and_one_launch(engine, pool, n, ring):
    """A lone Block-shaped group at each side of the threshold, at 668 records (N = 1,000) and at 6,668 (N = 10,000): verdicts equal the
    oracle and hs_verify_rec128, the counters show the kernel the threshold names, and the group is exactly one launch."""
    recs, _ = pool
    _committee(engine, recs)
    rng = np.random.default_rng(1000 + n)
    try:
        with engine.queue(ring_records=ring) as q:
            for _ in range(2):
                idx = rng.integers(0, len(recs), n)
                launches, d = _lone(engine, q, pool, idx, block_modes(n))
                assert launches == 1
                assert _routed(d, n, n >= BULK_MIN), d
    finally:
        _clear(engine)


def test_bulk_group_wraps_the_end_of_the_ring(engine, pool):
    """A bulk group whose records straddle the last ring slot: logical record i is slot (base + i) & mask."""
    recs, _ = pool
    ring = 4096 if BULK_MIN + 200 <= 2048 else 16384
    m = BULK_MIN + 200
    _committee(engine, recs)
    rng = np.random.default_rng(1100)
    try:
        with engine.queue(ring_records=ring) as q:
            filler = ring - m // 2                              # the next group starts m / 2 slots before the end
            _lone(engine, q, pool, rng.integers(0, len(recs), filler), block_modes(filler))
            for _ in range(2):                                  # the second one starts 37 slots further from the end
                idx = rng.integers(0, len(recs), m)
                launches, d = _lone(engine, q, pool, idx, block_modes(m))
                assert launches == 1 and _routed(d, m, True), d
                _lone(engine, q, pool, rng.integers(0, len(recs), ring - m - 37), block_modes(ring - m - 37))
    finally:
        _clear(engine)


def test_bulk_small_and_tiny_requests_from_8_threads(engine, pool):
    """8 threads each submit groups on both sides of the threshold, each followed by two 1..8-record requests, consumed by wait, poll
    and callback in turn; statuses are asserted here once every callback has fired.  Every bulk-size group is one bulk launch of its
    own; everything else rides in k_verify_small launches."""
    recs, _ = pool
    sizes = [BULK_MIN, 65, BULK_MIN + 333, BULK_MIN - 1, 1200] * 2
    _committee(engine, recs)
    try:
        with engine.queue(ring_records=16384) as q:
            s0 = q.stats()
            res = _run_group_threads(q, pool, sizes, 8, seed=1200)
            d = _delta(q.stats(), s0)
        _check(pool, res, 8 * len(sizes) * 3)
        bulk = [len(idx) for idx, *_ in res if len(idx) >= BULK_MIN]
        assert len(bulk) == 8 * sum(n >= BULK_MIN for n in sizes)
        assert d["bulk_launches"] == len(bulk) and d["bulk_records"] == sum(bulk), d
        assert d["small_records"] == sum(len(idx) for idx, *_ in res) - sum(bulk), d
        assert d["slow_requests"] == 0 and d["slow_records"] == 0, d
    finally:
        _clear(engine)


def test_small_requests_never_count_as_bulk_and_slow_groups_count_as_slow(engine, pool):
    """Without a committee every request takes the slow path, whatever its size.  With one, small requests and sub-threshold groups
    take k_verify_small and never count as bulk."""
    recs, _ = pool
    rng = np.random.default_rng(1300)
    _clear(engine)
    with engine.queue(ring_records=16384) as q:
        held = []
        for n in (3, 64, BULK_MIN - 1, BULK_MIN + 10):
            idx = rng.integers(0, len(recs), n)
            held.append((_submit(q, recs[idx], block_modes(n)), idx))
        for t, idx in held:
            assert (q.wait(t) == _expect(pool, idx, block_modes(len(idx)))).all()
        assert q.stats() == dict(small_launches=0, small_records=0, bulk_launches=0, bulk_records=0, slow_requests=4,
                                 slow_records=3 + 64 + 2 * BULK_MIN + 9)
    _committee(engine, recs)
    try:
        with engine.queue(ring_records=16384) as q:
            held = []
            for k in range(40):
                n = int(rng.integers(1, 65))
                idx = rng.integers(0, len(recs), n)
                mode = k % 2
                if k % 5 == 0:
                    n = max(1, BULK_MIN - 1 - k)
                    idx = rng.integers(0, len(recs), n)
                    held.append((_submit(q, recs[idx], block_modes(n)), idx, block_modes(n)))
                else:
                    held.append((q.submit(recs[idx], mode=mode), idx, np.full(n, mode, np.uint8)))
            for t, idx, modes in held:
                assert t is not None and (q.wait(t) == _expect(pool, idx, modes)).all()
            s = q.stats()
            assert s["bulk_launches"] == 0 and s["bulk_records"] == 0 and s["slow_requests"] == 0, s
            assert s["small_records"] == sum(len(idx) for _, idx, _ in held) and s["small_launches"] >= 1, s
    finally:
        _clear(engine)


def test_bulk_groups_across_committee_update(engine, oracle):
    """hs_committee_update with bulk groups in flight: they complete with the old committee's verdicts; a bulk group signed by the new
    validators afterwards takes the bulk kernel (one launch), and groups holding removed keys take the slow path."""
    g = BULK_MIN + 36
    w = make_workload(oracle, 6 * g, n_keys=64, seed=1400)
    recs = to_rec128(w)
    recs[::41, 3] ^= 0x20                                     # corrupted signatures (keys left intact: every key stays registered)
    modes = block_modes(g)
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    engine.committee_register(w["pks"])
    nw = make_workload(oracle, g, n_keys=8, seed=1401, corrupt_frac=0.0)
    new_recs = to_rec128(nw)
    try:
        with engine.queue(ring_records=16384) as q:
            s0 = q.stats()
            tickets = [(q.submit_group(recs[i:i + g], modes), i) for i in range(0, 6 * g, g)]
            assert all(t is not None for t, _ in tickets)
            engine.committee_update(add=nw["pks"], remove=np.arange(4, dtype=np.uint32))
            for t, i in tickets:
                assert (q.wait(t) == want[modes.astype(np.intp), np.arange(i, i + g)]).all()
            d = _delta(q.stats(), s0)                           # a group not yet dispatched when the update ran takes the slow path
            assert d["bulk_launches"] + d["slow_requests"] == 6 and d["bulk_records"] + d["slow_records"] == 6 * g, d
            l0, s1 = engine.kernel_launches, q.stats()
            assert q.wait(q.submit_group(new_recs, modes)).all()
            assert engine.kernel_launches - l0 == 1 and _routed(_delta(q.stats(), s1), g, True)
            s2 = q.stats()
            again = [(q.submit_group(recs[i:i + g], modes), i) for i in range(0, 6 * g, g)]   # every group holds a removed key
            for t, i in again:
                assert (q.wait(t) == want[modes.astype(np.intp), np.arange(i, i + g)]).all()
            d = _delta(q.stats(), s2)
            assert d["slow_requests"] == 6 and d["bulk_launches"] == 0, d
    finally:
        _clear(engine)


def test_bulk_teardown_fires_every_callback_once(oracle):
    """hs_queue_destroy and hs_ctx_destroy with bulk groups (and small requests) in flight: every callback fires once with the right
    verdicts, and no thread is left behind."""
    from hotstuff_b200 import Engine
    g = BULK_MIN + 100
    groups = min(8, 16000 // (g + 2))                         # every request fits the 16,384-record ring at once
    w = make_workload(oracle, groups * g, n_keys=32, seed=1500)
    recs = to_rec128(w)
    recs[::37, 9] ^= 0x04
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    e = Engine(0)
    try:
        e.committee_register(w["pks"])
        e.queue().close()                                     # lets the CUDA runtime settle its own threads
        for via_ctx in (False, True):
            before = _threads()
            q = e.queue(ring_records=16384)
            fired, lock = {}, threading.Lock()

            def cb(ticket, status, bits):
                with lock:
                    fired.setdefault(ticket, []).append((status, bits))

            expect = {}
            for i in range(0, groups * g, g):
                modes = block_modes(g)
                expect[q.submit_group(recs[i:i + g], modes, callback=cb)] = want[modes.astype(np.intp), np.arange(i, i + g)]
                expect[q.submit(recs[i + 1:i + 3], callback=cb)] = want[0, i + 1:i + 3]
            if via_ctx:
                q.h = None
                e._queues.remove(q)
                e.close()
            else:
                q.close()
            assert sorted(fired) == sorted(expect) and all(len(v) == 1 for v in fired.values())
            for t, v in fired.items():
                assert v[0][0] == 0 and (v[0][1] == expect[t]).all()
            assert _threads() == before
    finally:
        e.close()
