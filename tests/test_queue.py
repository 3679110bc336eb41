"""The verify queue (hs_queue_*, Engine.queue): concurrent small requests coalesced into shared launches of the latency kernel.
Every ticket's verdicts must equal hs_verify_rec128 on the same records and the oracle, whichever way the ticket is consumed."""
import os
import struct
import subprocess
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial, make_workload, to_rec128

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pool(oracle, golden):
    """Golden vectors (32-byte messages), randomised adversarial records and honest / corrupted records, with both oracle verdicts."""
    vs = [v for v in golden["vectors"] if len(v["msg"]) == 64]
    gold = np.array([np.frombuffer(bytes.fromhex(v["sig"] + v["pk"] + v["msg"]), np.uint8) for v in vs])
    w = make_workload(oracle, 2000, n_keys=40, seed=7100, corrupt_frac=0.1)
    recs = np.concatenate([gold, make_adversarial(oracle, 3000, seed=7101), to_rec128(w)], axis=0)
    return recs, (oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1))


def _requests(rng, n_pool, count):
    return [(rng.integers(0, n_pool, int(rng.integers(1, 9))), int(rng.integers(0, 2))) for _ in range(count)]


def _run_threads(q, pool, n_threads, per_thread, seed):
    """n_threads Python threads each submit per_thread requests (1..8 records, mixed modes) and consume them by wait, poll
    and callback in turn.  Returns [(record indices, mode, verdicts)]."""
    recs, _ = pool
    out, errors, lock = [], [], threading.Lock()

    def worker(t):
        rng = np.random.default_rng(seed + t)
        reqs = _requests(rng, len(recs), per_thread)
        try:
            for lo in range(0, per_thread, 48):
                held = []
                for k, (idx, mode) in enumerate(reqs[lo:lo + 48]):
                    how = (lo + k) % 3
                    cb = None
                    if how == 2:
                        def cb(ticket, status, bits, idx=idx, mode=mode):
                            assert status == 0
                            with lock:
                                out.append((idx, mode, bits))
                    while True:
                        ticket = q.submit(recs[idx], mode=mode, callback=cb)
                        if ticket is not None:
                            break
                        threading.Event().wait(0.0005)   # ring full: back-pressure
                    held.append((ticket, how, idx, mode))
                for ticket, how, idx, mode in held:
                    if how == 0:
                        bits = q.wait(ticket)
                    elif how == 1:
                        bits = q.poll(ticket)
                        while bits is None:
                            bits = q.poll(ticket)
                    else:
                        continue
                    with lock:
                        out.append((idx, mode, bits))
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))

    ts = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[:3]
    return out


def _check(engine, pool, results, expect):
    recs, want = pool
    assert len(results) == expect
    for idx, mode, bits in results:
        assert (bits == want[mode][idx]).all(), (idx, mode)
        assert (bits == engine.verify_rec128(recs[idx], mode=mode)).all(), (idx, mode)


def test_queue_parity_registered_committee(engine, pool):
    """8 threads x 2,000 requests against a committee that includes the adversarial keys: device path, every consumption kind."""
    recs, _ = pool
    engine.committee_register(np.unique(recs[:, 64:96], axis=0))
    try:
        l0 = engine.kernel_launches
        with engine.queue() as q:
            res = _run_threads(q, pool, 8, 2000, seed=11)
        assert engine.kernel_launches - l0 < 16000            # requests shared launches
        _check(engine, pool, res, 16000)
    finally:
        engine.committee_register(np.zeros((0, 32), np.uint8))


def test_queue_fallback_without_committee_and_outside_it(engine, pool):
    """No committee (key-cache path) and a committee holding only some of the keys: the slow path gives the same verdicts."""
    recs, _ = pool
    engine.committee_register(np.zeros((0, 32), np.uint8))
    with engine.queue() as q:
        res = _run_threads(q, pool, 4, 300, seed=21)
    _check(engine, pool, res, 1200)
    keys = np.unique(recs[:, 64:96], axis=0)
    engine.committee_register(keys[::2])
    try:
        with engine.queue() as q:
            res = _run_threads(q, pool, 4, 300, seed=31)
        _check(engine, pool, res, 1200)
    finally:
        engine.committee_register(np.zeros((0, 32), np.uint8))


def test_queue_ring_wrap_and_back_pressure(engine, pool):
    """A 256-record ring: submit until it is full (None), drain, continue — verdicts stay right across many wraps.  Ring space is
    released when a request completes, so requests of 33..64 records are used: they arrive faster than two launches retire."""
    recs, want = pool
    engine.committee_register(np.unique(recs[:, 64:96], axis=0))
    rng = np.random.default_rng(41)
    try:
        with engine.queue(ring_records=200) as q:                 # rounded up to 256
            full_seen, done = 0, 0
            while full_seen < 20:
                held = []
                while True:
                    idx = rng.integers(0, len(recs), int(rng.integers(33, 65)))
                    ticket = q.submit(recs[idx])
                    if ticket is None:
                        full_seen += 1
                        break
                    held.append((ticket, idx))
                    assert len(held) < 5000, "the ring never filled"
                assert sum(len(i) for _, i in held) > 256 - 64     # it filled up
                for ticket, idx in held:
                    assert (q.wait(ticket) == want[0][idx]).all()
                    done += len(idx)
            assert done > 20 * 192                                  # many wraps of the 256-record ring
    finally:
        engine.committee_register(np.zeros((0, 32), np.uint8))


def _burst_file(oracle, tmp_path, n):
    w = make_workload(oracle, n, n_keys=64, seed=5151, corrupt_frac=0.01)
    recs = to_rec128(w)
    want = oracle.verify_rec128(recs).astype(np.uint8)
    path = tmp_path / "burst.bin"
    path.write_bytes(struct.pack("<I", 64) + w["pks"].tobytes() + struct.pack("<I", n) + recs.tobytes() + want.tobytes())
    return str(path)


def test_queue_coalesces_a_native_burst(engine, oracle, tmp_path):
    """4,096 single-record requests from 8 native threads (tests/cpp/queue_burst.cpp): at most two launches are in flight and a
    launch cannot finish before R's square-root chain, so the burst must average >= 4 records per queue launch.  The same burst
    through hs::VerifyQueue (std::future per request) must also verify."""
    import json
    from hotstuff_b200 import build
    lib = build.build_engine()
    exe = str(tmp_path / "queue_burst")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-o", exe, os.path.join(ROOT, "tests", "cpp", "queue_burst.cpp"), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    path = _burst_file(oracle, tmp_path, 4096)
    for extra in ([], ["--hpp"]):
        out = subprocess.run([exe, path, "8"] + extra, capture_output=True, text=True)
        assert out.returncode == 0, out.stdout + out.stderr
        r = json.loads(out.stdout.strip().splitlines()[-1])
        assert r["mismatches"] == 0 and r["records"] == 4096
        if not extra:
            assert r["records_per_launch"] >= 4.0, r


def test_queue_beside_a_large_synchronous_verify(engine, oracle, pool):
    """A 2^16-record hs_verify_rec128 in another thread while the queue is busy: both sets of results are right."""
    recs, want = pool
    engine.committee_register(np.unique(recs[:, 64:96], axis=0))
    big = np.tile(recs[:4096], (16, 1))
    big_want = np.tile(want[0][:4096], 16)
    got_big = []
    try:
        with engine.queue() as q:
            t = threading.Thread(target=lambda: got_big.append(engine.verify_rec128(big)))
            t.start()
            res = _run_threads(q, pool, 4, 600, seed=51)
            t.join()
        assert len(got_big) == 1 and (got_big[0] == big_want).all()
        _check(engine, pool, res, 2400)
    finally:
        engine.committee_register(np.zeros((0, 32), np.uint8))


def test_queue_sees_committee_updates(engine, oracle):
    """hs_committee_update with requests in flight: they complete correctly, and requests submitted after the update are
    judged against the new committee (new validators verify on the device path; removed keys are unregistered)."""
    w = make_workload(oracle, 600, n_keys=24, seed=6161, corrupt_frac=0.05)
    recs = to_rec128(w)
    want = oracle.verify_rec128(recs)
    engine.committee_register(w["pks"])
    seeds = np.random.default_rng(62).integers(0, 256, (4, 32), dtype=np.uint8)
    newpk = oracle.keygen_batch(seeds)
    m = np.random.default_rng(63).integers(0, 256, (4, 32), dtype=np.uint8)
    sg = oracle.sign_batch(seeds, newpk, np.arange(4, dtype=np.uint32), m.reshape(-1), np.arange(5, dtype=np.uint64) * 32)
    new_recs = np.concatenate([sg, newpk, m], axis=1)
    try:
        with engine.queue() as q:
            tickets = [(q.submit(recs[i:i + 3]), i) for i in range(0, 600, 3)]
            engine.committee_update(add=newpk, remove=np.arange(4, dtype=np.uint32))
            for t, i in tickets:                                   # in flight across the update
                assert (q.wait(t) == want[i:i + 3]).all()
            l0 = engine.kernel_launches
            after = [q.submit(new_recs[i:i + 1]) for i in range(4)]
            assert all(q.wait(t).all() for t in after)
            assert engine.kernel_launches - l0 <= 4                # device path: no generic-pass launches
            again = [(q.submit(recs[i:i + 3]), i) for i in range(0, 600, 3)]   # removed keys now take the slow path
            for t, i in again:
                assert (q.wait(t) == want[i:i + 3]).all()
    finally:
        engine.committee_register(np.zeros((0, 32), np.uint8))


def _threads():
    return len(os.listdir("/proc/self/task"))


def test_queue_teardown_fires_every_callback_once(oracle):
    """hs_queue_destroy and hs_ctx_destroy with requests in flight: every callback fires exactly once and no thread is left."""
    from hotstuff_b200 import Engine
    w = make_workload(oracle, 512, n_keys=16, seed=7171, corrupt_frac=0.05)
    recs = to_rec128(w)
    want = oracle.verify_rec128(recs)
    e = Engine(0)
    try:
        e.committee_register(w["pks"])
        e.queue().close()                         # first queue of the process: lets the CUDA runtime settle its own threads
        for via_ctx in (False, True):
            before = _threads()
            q = e.queue()
            fired, lock = {}, threading.Lock()

            def cb(ticket, status, bits):
                with lock:
                    fired.setdefault(ticket, []).append((status, bits))

            ticket_idx = {}
            for i in range(0, 512, 2):
                ticket_idx[q.submit(recs[i:i + 2], callback=cb)] = slice(i, i + 2)
            if via_ctx:                           # hs_ctx_destroy tears down the queue still attached to it
                q.h = None
                e._queues.remove(q)
                e.close()
            else:
                q.close()
            assert sorted(fired) == sorted(ticket_idx) and all(len(v) == 1 for v in fired.values())
            for t, v in fired.items():
                assert v[0][0] == 0 and (v[0][1] == want[ticket_idx[t]]).all()
            assert _threads() == before
    finally:
        e.close()


def test_queue_misuse_is_an_argument_error(engine, oracle):
    from hotstuff_b200 import EngineError
    w = make_workload(oracle, 70, n_keys=4, seed=8181)
    recs = to_rec128(w)
    with engine.queue() as q:
        t = q.submit(recs[:2])
        assert q.wait(t).all()
        with pytest.raises(EngineError, match="status 2"):
            q.wait(t)                              # read twice
        with pytest.raises(EngineError, match="status 2"):
            q.poll(t)
        got = []
        t = q.submit(recs[:1], callback=lambda *a: got.append(a))
        with pytest.raises(EngineError, match="status 2"):
            q.wait(t)                              # a callback ticket is not readable
        for bad_n in (recs[:0], recs[:65]):
            with pytest.raises(EngineError, match="status 2"):
                q.submit(bad_n)
        with pytest.raises(EngineError, match="status 2"):
            q.submit(recs[:1], mode=2)
