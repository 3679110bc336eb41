"""Whole certificates through the verify queue (hs_queue_submit_group, VerifyQueue.submit_group): one request per consensus message,
up to the ring's capacity, a verdict mode per record.  Record i's verdict must equal hs_verify_rec128 on that record in its mode and
the oracle, on the device path and the slow path, whichever way the ticket is consumed."""
import os
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial, make_workload, to_rec128

pytestmark = pytest.mark.gpu
RING = 4096


@pytest.fixture(scope="module")
def pool(oracle, golden, engine):
    """Golden, adversarial and honest / corrupted records with the oracle's and the engine's (hs_verify_rec128) verdicts per mode."""
    vs = [v for v in golden["vectors"] if len(v["msg"]) == 64]
    gold = np.array([np.frombuffer(bytes.fromhex(v["sig"] + v["pk"] + v["msg"]), np.uint8) for v in vs])
    w = make_workload(oracle, 3000, n_keys=48, seed=9100, corrupt_frac=0.05)
    recs = np.concatenate([gold, make_adversarial(oracle, 2000, seed=9101), to_rec128(w)], axis=0)
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    eng = np.stack([engine.verify_rec128(recs, mode=0), engine.verify_rec128(recs, mode=1)])
    assert (want == eng).all()
    return recs, want


def block_modes(n):
    """The shape of a Block: author signature strict, then the QC's votes batch-eq, then the TC's votes strict."""
    m = np.zeros(n, np.uint8)
    m[1:1 + (2 * n) // 3] = 1
    return m


def _expect(pool, idx, modes):
    return pool[1][modes.astype(np.intp), idx]


def _committee(engine, recs):
    engine.committee_register(np.unique(recs[:, 64:96], axis=0))


def _clear(engine):
    engine.committee_register(np.zeros((0, 32), np.uint8))


def _submit(q, recs, modes, callback=None):
    while True:
        t = q.submit_group(recs, modes, callback=callback)
        if t is not None:
            return t
        threading.Event().wait(0.0005)  # ring full: back-pressure


def _run_group_threads(q, pool, sizes, n_threads, seed):
    """n_threads threads each submit a group of every size in `sizes` (Block-shaped modes) interleaved with small requests, and
    consume them by wait, poll and callback in turn.  Returns [(indices, modes, status, verdicts)] once every request has been
    consumed: the waited and polled ones by their threads, the callback ones when their callbacks have fired.  A callback only
    records its status (an assert inside a ctypes callback would be swallowed); _check asserts on it."""
    recs, _ = pool
    out, errors = [], []
    cv = threading.Condition()
    pending_cb = [0]

    def worker(t):
        rng = np.random.default_rng(seed + t)
        try:
            held = []
            for k, n in enumerate(sizes):
                how = (k + t) % 3
                for kind in ("group", "small", "small"):
                    if kind == "group":
                        idx, modes = rng.integers(0, len(recs), n), block_modes(n)
                    else:
                        idx = rng.integers(0, len(recs), int(rng.integers(1, 9)))
                        modes = np.full(len(idx), int(rng.integers(0, 2)), np.uint8)
                    cb = None
                    if how == 2:
                        def cb(ticket, status, bits, idx=idx, modes=modes):
                            with cv:
                                out.append((idx, modes, status, bits))
                                pending_cb[0] -= 1
                                cv.notify_all()
                        with cv:
                            pending_cb[0] += 1       # counted before the submit: the callback may fire before it returns
                    if kind == "group":
                        ticket = _submit(q, recs[idx], modes, cb)
                    else:
                        while (ticket := q.submit(recs[idx], mode=int(modes[0]), callback=cb)) is None:
                            threading.Event().wait(0.0005)
                    held.append((ticket, how, idx, modes))
            for ticket, how, idx, modes in held:
                if how == 0:
                    bits = q.wait(ticket)
                elif how == 1:
                    while (bits := q.poll(ticket)) is None:
                        pass
                else:
                    continue
                with cv:
                    out.append((idx, modes, 0, bits))   # wait / poll raise on a non-zero status
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))

    ts = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[:3]
    with cv:
        assert cv.wait_for(lambda: pending_cb[0] == 0, timeout=300), "%d callbacks never fired" % pending_cb[0]
        return list(out)


def _check(pool, results, expect):
    assert len(results) == expect
    for idx, modes, status, bits in results:
        assert status == 0
        assert len(bits) == len(idx)
        assert (bits == _expect(pool, idx, modes)).all(), (len(idx), np.flatnonzero(bits != _expect(pool, idx, modes))[:8])


def test_group_parity_device_path_from_8_threads(engine, pool):
    """Groups of 1, 64, 65 and 668 records (Block-shaped modes) from 8 threads, interleaved with small requests, then one group of
    the ring's whole capacity on a fresh queue: every verdict equals the oracle and hs_verify_rec128 in that record's mode."""
    recs, _ = pool
    _committee(engine, recs)
    try:
        with engine.queue(ring_records=RING) as q:
            res = _run_group_threads(q, pool, [1, 64, 65, 668] * 2, 8, seed=100)
        _check(pool, res, 8 * 8 * 3)                          # after close: every callback has fired
        with engine.queue(ring_records=RING) as q:
            idx = np.random.default_rng(101).integers(0, len(recs), RING)
            modes = block_modes(RING)
            bits = q.wait(_submit(q, recs[idx], modes))
        _check(pool, [(idx, modes, 0, bits)], 1)
    finally:
        _clear(engine)


def test_group_verdict_is_hs_verify_rec128_per_record(engine, pool):
    """The per-record contract, literally: record i of a group equals hs_verify_rec128(&recs[i], 1, modes[i])."""
    recs, _ = pool
    rng = np.random.default_rng(102)
    idx = rng.integers(0, len(recs), 96)
    modes = rng.integers(0, 2, 96).astype(np.uint8)
    single = np.array([engine.verify_rec128(recs[i:i + 1], mode=int(m))[0] for i, m in zip(idx, modes)])
    _committee(engine, recs)
    try:
        with engine.queue() as q:
            assert (q.wait(_submit(q, recs[idx], modes)) == single).all()
    finally:
        _clear(engine)
    with engine.queue() as q:                                  # slow path
        assert (q.wait(_submit(q, recs[idx], modes)) == single).all()


def test_group_slow_path_without_committee_and_with_a_missing_key(engine, oracle, pool):
    """No committee: every group takes the slow path.  A committee missing one key of a group: that group takes the slow path
    while groups between it keep the device path; verdicts are the same either way."""
    _clear(engine)
    with engine.queue() as q:
        res = _run_group_threads(q, pool, [1, 65, 668], 4, seed=200)
    _check(pool, res, 4 * 3 * 3)
    w = make_workload(oracle, 2000, n_keys=32, seed=9200, corrupt_frac=0.05)
    recs = to_rec128(w)
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    missing = w["key_idx"][0]
    engine.committee_register(np.delete(w["pks"], missing, axis=0))
    try:
        with engine.queue() as q:
            held = []
            for k in range(12):
                lo = (k * 150) % (2000 - 668)
                idx = np.arange(lo, lo + 668)
                if k % 2:
                    idx = idx[w["key_idx"][idx] != missing]      # device path
                else:
                    idx[5] = 0                                   # record 0 has the missing key: slow path
                modes = block_modes(len(idx))
                held.append((_submit(q, recs[idx], modes), idx, modes))
            for t, idx, modes in held:
                assert (q.wait(t) == want[modes.astype(np.intp), idx]).all()
    finally:
        _clear(engine)


def test_group_misuse_is_an_argument_error(engine, pool):
    from hotstuff_b200 import EngineError
    recs, _ = pool
    with engine.queue(ring_records=1024) as q:
        for bad in (recs[:0], recs[:1025]):
            with pytest.raises(EngineError, match="status 2"):
                q.submit_group(bad)
        modes = np.zeros(10, np.uint8)
        modes[7] = 2
        with pytest.raises(EngineError, match="status 2"):
            q.submit_group(recs[:10], modes)
        with pytest.raises(ValueError):
            q.submit_group(recs[:10], modes[:9])
        t = q.submit_group(recs[:1024])                         # exactly the capacity is fine
        assert len(q.wait(t)) == 1024


def test_group_back_pressure_then_success(engine, pool):
    """668-record groups on a 1,024-record ring: the second one finds no room (None) while the first is in flight; after draining, the
    same group is accepted and verified."""
    recs, want = pool
    _committee(engine, recs)
    rng = np.random.default_rng(300)
    try:
        with engine.queue(ring_records=1024) as q:
            for _ in range(3):
                held, full = [], False
                for _ in range(50):
                    idx = rng.integers(0, len(recs), 668)
                    t = q.submit_group(recs[idx], block_modes(668))
                    if t is None:
                        full = True
                        break
                    held.append((t, idx))
                assert full and held
                for t, idx in held:
                    assert (q.wait(t) == _expect(pool, idx, block_modes(668))).all()
                t = q.submit_group(recs[idx], block_modes(668))
                assert t is not None and (q.wait(t) == _expect(pool, idx, block_modes(668))).all()
    finally:
        _clear(engine)


def test_lone_device_group_is_one_launch(engine, oracle):
    """A 668-record Block (1 author + 667 QC votes of a 1,000-validator committee) with every key registered and nothing else
    pending costs exactly one launch."""
    w = make_workload(oracle, 668, n_keys=1000, seed=9400)
    recs = to_rec128(w)
    recs[::100, 17] ^= 0x08                                    # 1 % corrupted signatures (the keys stay registered ones)
    modes = block_modes(668)
    want = np.where(modes == 1, oracle.verify_rec128(recs, mode=1), oracle.verify_rec128(recs, mode=0))
    engine.committee_register(w["pks"])
    try:
        with engine.queue() as q:
            for _ in range(3):
                l0 = engine.kernel_launches
                bits = q.wait(q.submit_group(recs, modes))
                assert engine.kernel_launches - l0 == 1
                assert (bits == want).all()
    finally:
        _clear(engine)


def test_groups_across_committee_update(engine, oracle):
    """hs_committee_update with groups in flight: they complete correctly; groups submitted after it are judged against the new
    committee (a group signed by new validators takes the device path: one launch)."""
    w = make_workload(oracle, 2000, n_keys=64, seed=9500, corrupt_frac=0.05)
    recs = to_rec128(w)
    modes = block_modes(200)
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    engine.committee_register(w["pks"])
    nw = make_workload(oracle, 200, n_keys=8, seed=9501, corrupt_frac=0.0)
    new_recs = to_rec128(nw)
    try:
        with engine.queue() as q:
            tickets = [(q.submit_group(recs[i:i + 200], modes), i) for i in range(0, 2000, 200)]
            engine.committee_update(add=nw["pks"], remove=np.arange(4, dtype=np.uint32))
            for t, i in tickets:
                assert (q.wait(t) == want[modes.astype(np.intp), np.arange(i, i + 200)]).all()
            l0 = engine.kernel_launches
            assert q.wait(q.submit_group(new_recs, modes)).all()
            assert engine.kernel_launches - l0 == 1
            again = [(q.submit_group(recs[i:i + 200], modes), i) for i in range(0, 2000, 200)]   # removed keys: slow path
            for t, i in again:
                assert (q.wait(t) == want[modes.astype(np.intp), np.arange(i, i + 200)]).all()
    finally:
        _clear(engine)


def test_large_slow_group_never_rides_in_a_launch(engine, oracle):
    """A slow-path request of more than 64 records between two device requests splits the dispatch: device group, large slow group,
    device group cost two queue launches plus the slow group's own synchronous launches, never one launch whose grid spans the slow
    group's records.  A large slow-path group first keeps the dispatcher busy, so the three are pending together and taken by one
    dispatch.  Every other grouping also costs two launches, so the count is exact whatever the timing."""
    w = make_workload(oracle, 6000, n_keys=64, seed=9700)
    recs = to_rec128(w)
    recs[::41, 3] ^= 0x20
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    engine.committee_register(w["pks"][1:])                   # key 0 unregistered: a group holding it takes the slow path
    dev = np.flatnonzero(w["key_idx"] != 0)
    a_idx, b_idx = dev[:300], dev[300:600]
    s_idx = np.arange(1000, 1300)                             # holds key 0 (every 64th record)
    h_idx = np.arange(1500, 1500 + 4096)

    def launches(q, idx):
        l0 = engine.kernel_launches
        modes = block_modes(len(idx))
        assert (q.wait(_submit(q, recs[idx], modes)) == want[modes.astype(np.intp), idx]).all()
        return engine.kernel_launches - l0

    try:
        with engine.queue(ring_records=16384) as q:
            assert launches(q, a_idx) == 1 and launches(q, b_idx) == 1
            l_s, l_h = launches(q, s_idx), launches(q, h_idx)
            assert launches(q, s_idx) == l_s and launches(q, h_idx) == l_h   # the slow path's launch count is fixed
            for _ in range(3):
                l0 = engine.kernel_launches
                tickets = [(_submit(q, recs[h_idx], block_modes(len(h_idx))), h_idx)]
                threading.Event().wait(0.0005)                 # the dispatcher is now inside the hold group's slow path
                tickets += [(_submit(q, recs[i], block_modes(len(i))), i) for i in (a_idx, s_idx, b_idx)]
                for t, i in tickets:
                    modes = block_modes(len(i))
                    assert (q.wait(t) == want[modes.astype(np.intp), i]).all()
                assert engine.kernel_launches - l0 == l_h + l_s + 2
    finally:
        _clear(engine)


def _threads():
    return len(os.listdir("/proc/self/task"))


def test_group_teardown_fires_every_callback_once(oracle):
    """hs_queue_destroy and hs_ctx_destroy with groups (and small requests) in flight: every callback fires once, with the right
    verdicts, and no thread is left.  Half of the groups hold key 0, which is not registered (slow path); the other half leave
    it out and take the device path, so their launches can still be in flight when the queue goes."""
    from hotstuff_b200 import Engine
    w = make_workload(oracle, 2048, n_keys=32, seed=9600)
    recs = to_rec128(w)
    recs[::37, 9] ^= 0x04                                     # corrupted signatures (keys left intact: registered keys stay registered)
    want = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    e = Engine(0)
    try:
        e.committee_register(w["pks"][1:])                    # key 0 unregistered
        e.queue().close()                                     # lets the CUDA runtime settle its own threads
        for via_ctx in (False, True):
            before = _threads()
            q = e.queue(ring_records=8192)
            fired, lock = {}, threading.Lock()

            def cb(ticket, status, bits):
                with lock:
                    fired.setdefault(ticket, []).append((status, bits))

            expect = {}
            for k, i in enumerate(range(0, 2048, 256)):
                idx = np.arange(i, i + 256)
                if k % 2:                                     # device path: the records of key 0 left out; the last group is one
                    idx = idx[w["key_idx"][idx] != 0]
                modes = block_modes(len(idx))
                expect[q.submit_group(recs[idx], modes, callback=cb)] = want[modes.astype(np.intp), idx]
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
