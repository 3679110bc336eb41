"""The verify queue's generic-key device path (hs_queue_generic, VerifyQueue.generic): with it on, a request the committee path
cannot serve (no committee registered, or a key outside it) is verified by k_queue_generic on the GPU instead of synchronously on
the dispatcher thread.  Every verdict must equal the oracle's, hs_verify_rec128's and the same request's on a queue with the option
off; the counters show which path each request took."""
import hashlib
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial
from test_queue_msgs import K, _clear, _register, make_req, want

pytestmark = pytest.mark.gpu
BULK_MIN = 1002


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(8100)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture(scope="module")
def foreign(oracle):
    """64 keys that are never registered."""
    rng = np.random.default_rng(8101)
    seeds = rng.integers(0, 256, size=(64, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture()
def no_committee(engine):
    _clear(engine)
    yield
    _clear(engine)


@pytest.fixture()
def committee(engine, keys):
    _register(engine, keys[1])
    yield
    _clear(engine)


def golden_recs(golden):
    vs = [v for v in golden["vectors"] if len(v["msg"]) == 64]
    return np.array([np.frombuffer(bytes.fromhex(v["sig"] + v["pk"] + v["msg"]), np.uint8) for v in vs])


def signed(oracle, keys, n, rng, corrupt=0.05):
    """n (sig | pk | msg) records over random Digests by random keys of `keys`; `corrupt` of them get a flipped bit in the
    signature or the Digest (never in the key, so a committee key stays registered)."""
    seeds, pks = keys
    kidx = rng.integers(0, len(pks), n).astype(np.uint32)
    msgs = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sig = oracle.sign_batch(seeds, pks, kidx, msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    recs = np.concatenate([sig, pks[kidx], msgs], axis=1)
    for i in np.flatnonzero(rng.random(n) < corrupt):
        b = int(rng.integers(0, 96))
        recs[i, b if b < 64 else b + 32] ^= 1 << int(rng.integers(0, 8))
    return recs


def oracle_bits(oracle, recs, modes):
    w = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    return w[np.asarray(modes, np.intp), np.arange(len(recs))]


def sync_bits(engine, recs, modes):
    """hs_verify_rec128 per record in its mode (one call per mode)."""
    out = np.zeros(len(recs), bool)
    for m in (0, 1):
        sel = np.flatnonzero(np.asarray(modes) == m)
        if len(sel):
            out[sel] = engine.verify_rec128(recs[sel], mode=m)
    return out


def retry(fn):
    while (t := fn()) is None:
        threading.Event().wait(0.0005)  # no room now: back-pressure
    return t


def submit_any(q, recs, modes, callback=None):
    """A small request through submit when it has one mode and at most 64 records, else through submit_group."""
    if len(recs) <= 64 and (modes == modes[0]).all():
        return retry(lambda: q.submit(recs, mode=int(modes[0]), callback=callback))
    return retry(lambda: q.submit_group(recs, modes, callback=callback))


def mixed_requests(oracle, keys, foreign, rng, sizes, foreign_frac):
    """Requests of the given sizes over committee keys; in `foreign_frac` of them one record (or more) is by a foreign key.  Modes
    are mixed per record in groups, one per small request."""
    reqs = []
    for n in sizes:
        recs = signed(oracle, keys, n, rng)
        if rng.random() < foreign_frac:
            k = int(rng.integers(1, max(2, n // 8) + 1))
            at = rng.choice(n, size=min(k, n), replace=False)
            recs[at] = signed(oracle, foreign, len(at), rng)
        modes = (rng.integers(0, 2, n) if n > 64 or rng.random() < 0.3 else np.full(n, int(rng.integers(0, 2)))).astype(np.uint8)
        reqs.append((recs, modes))
    return reqs


def test_no_committee_every_request_takes_the_generic_path(engine, oracle, golden, keys, no_committee):
    """No committee registered: the golden vectors (the speccheck classes among them) and adversarial records (non-canonical S,
    small-order and non-decompressible A / R, mixed-order keys, bit flips) through submit, submit_group with mixed modes and
    submit_msgs.  Every request takes k_queue_generic; none runs on the dispatcher thread, and no small launch is made."""
    rng = np.random.default_rng(1)
    recs = np.concatenate([golden_recs(golden), make_adversarial(oracle, 900, seed=8102), signed(oracle, keys, 200, rng)])
    reqs, lo = [], 0
    sizes = [1, 2, 5, 31, 64, 64, 3, 200, 1, 7, 130, 64]
    while lo < len(recs):
        n = sizes[len(reqs) % len(sizes)]
        chunk = recs[lo:lo + n]
        modes = rng.integers(0, 2, len(chunk)).astype(np.uint8) if len(chunk) > 64 else np.full(len(chunk), len(reqs) % 2, np.uint8)
        reqs.append((chunk, modes))
        lo += n
    msgs = [make_req(oracle, keys, shape, n, rng, corrupt=0.1) for shape, n in (("vote", 3), ("timeout", 40), ("tc", 67), ("block_tc", 300))]
    # the golden vectors' messages as preimages: the records are judged over their SHA-512 Digests
    vs = golden["vectors"]
    pres = [bytes.fromhex(v["msg"]) for v in vs]
    off = np.zeros(len(pres) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in pres])
    msgs.append(dict(pre=np.frombuffer(b"".join(pres), np.uint8), off=off,
                     sig=np.array([np.frombuffer(bytes.fromhex(v["sig"]), np.uint8) for v in vs]),
                     pk=np.array([np.frombuffer(bytes.fromhex(v["pk"]), np.uint8) for v in vs]),
                     mi=np.arange(len(vs), dtype=np.uint32), modes=(np.arange(len(vs)) % 2).astype(np.uint8)))
    with engine.queue(ring_records=4096) as q:
        q.generic(True)
        t_recs = [submit_any(q, r, m) for r, m in reqs]
        t_msgs = [retry(lambda r=r: q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"])) for r in msgs]
        for (r, m), t in zip(reqs, t_recs):
            bits = q.wait(t)
            w = oracle_bits(oracle, r, m)
            assert (bits == w).all(), np.flatnonzero(bits != w)[:8]
            assert (bits == sync_bits(engine, r, m)).all()
        for r, t in zip(msgs, t_msgs):
            bits = q.wait(t)
            w = want(oracle, r)
            assert (bits == w).all(), np.flatnonzero(bits != w)[:8]
        g, s, d = q.generic_stats(), q.stats(), q.digest_stats()
    n_req = len(reqs) + len(msgs)
    assert g["requests"] == n_req
    assert g["records"] == sum(len(r) for r, _ in reqs) + sum(len(r["mi"]) for r in msgs)
    assert 1 <= g["launches"] <= n_req
    assert s["slow_requests"] == 0 and s["slow_records"] == 0
    assert s["small_launches"] == 0 and s["bulk_launches"] == 0
    assert d["msgs_requests"] == len(msgs) and 1 <= d["digest_launches"] <= len(msgs)


def test_option_off_is_the_slow_path_and_toggling_restores_it(engine, oracle, keys, foreign, no_committee):
    rng = np.random.default_rng(2)
    recs = signed(oracle, foreign, 40, rng)
    with engine.queue(ring_records=256) as q:
        assert (q.wait(q.submit(recs[:8], mode=1)) == oracle.verify_rec128(recs[:8], mode=1)).all()
        assert q.stats()["slow_requests"] == 1 and q.generic_stats()["requests"] == 0
        q.generic(True)
        assert (q.wait(q.submit(recs[8:16], mode=0)) == oracle.verify_rec128(recs[8:16], mode=0)).all()
        assert q.stats()["slow_requests"] == 1 and q.generic_stats() == dict(launches=1, records=8, requests=1)
        # turned off with requests in flight: they complete, and later requests take the slow path again
        tickets = [q.submit(recs[16 + 4 * i:20 + 4 * i], mode=i % 2) for i in range(4)]
        q.generic(False)
        for i, t in enumerate(tickets):
            assert (q.wait(t) == oracle.verify_rec128(recs[16 + 4 * i:20 + 4 * i], mode=i % 2)).all()
        s0 = q.stats()["slow_requests"]
        assert (q.wait(q.submit(recs[32:40], mode=0)) == oracle.verify_rec128(recs[32:40], mode=0)).all()
        assert q.stats()["slow_requests"] == s0 + 1
        assert q.generic_stats()["requests"] + s0 == 1 + 1 + 4


@pytest.mark.parametrize("ring,sizes", [
    (64, [1, 3, 7, 17, 33, 64, 5, 1, 2, 40, 64, 9, 23, 64, 1, 11] * 3),  # every small size, wrapping a 64-record ring many times
    (2048, [65, 300, 1, 64, BULK_MIN, 7, 200, BULK_MIN + 40, 3, 640, 64, 1]),  # groups over 64 and over the bulk cut-over
])
def test_committee_with_foreign_keys_matches_the_option_off_queue(engine, oracle, keys, foreign, committee, ring, sizes):
    """Requests mixing registered and unregistered keys, interleaved with device requests, with records wrapping the ring's end:
    verdicts equal the oracle's and those of the same requests on a queue with the option off.  Only the requests with a
    foreign key take the generic path; the others keep the small and bulk launches."""
    rng = np.random.default_rng(3 + ring)
    reqs = mixed_requests(oracle, keys, foreign, rng, sizes, foreign_frac=0.4)
    registered = set(map(bytes, keys[1]))
    n_foreign = sum(1 for r, _ in reqs if set(map(bytes, r[:, 64:96])) - registered)
    with engine.queue(ring_records=ring) as q, engine.queue(ring_records=ring) as plain:
        q.generic(True)
        for rep in range(2):  # the second pass starts wherever the first left the ring
            tickets = [submit_any(q, r, m) for r, m in reqs]
            got = [q.wait(t) for t in tickets]
            for (r, m), bits in zip(reqs, got):
                w = oracle_bits(oracle, r, m)
                assert (bits == w).all(), np.flatnonzero(bits != w)[:8]
                assert (bits == plain.wait(submit_any(plain, r, m))).all()
        g, s = q.generic_stats(), q.stats()
        assert s["slow_requests"] == 0
        assert g["requests"] == 2 * n_foreign and n_foreign > 0
        assert s["small_launches"] > 0
        assert plain.stats()["slow_requests"] == 2 * n_foreign and plain.generic_stats()["requests"] == 0


def test_sixteen_threads_callbacks_and_poll_wait(engine, oracle, keys, foreign, committee):
    """16 threads submit mixed requests (registered, foreign and mixed keys) with callbacks and with poll / wait: every ticket
    completes exactly once with the oracle's verdicts."""
    rng = np.random.default_rng(4)
    per = [mixed_requests(oracle, keys, foreign, np.random.default_rng(400 + t), list(rng.choice([1, 2, 5, 30, 64, 90, 300], 12)), 0.5)
           for t in range(16)]
    errors, seen, lock = [], {}, threading.Lock()
    with engine.queue(ring_records=1024) as q:
        q.generic(True)

        def worker(t):
            try:
                done = threading.Semaphore(0)
                pending = []
                for i, (r, m) in enumerate(per[t]):
                    w = oracle_bits(oracle, r, m)
                    if i % 2:
                        def cb(ticket, status, bits, w=w, key=(t, i)):
                            with lock:
                                seen[key] = seen.get(key, 0) + 1
                            if status != 0 or not (bits == w).all():
                                errors.append((key, status))
                            done.release()
                        submit_any(q, r, m, callback=cb)
                        pending.append(None)
                    else:
                        tk = submit_any(q, r, m)
                        if i % 4 == 0:
                            while (bits := q.poll(tk)) is None:
                                threading.Event().wait(0.0002)
                        else:
                            bits = q.wait(tk)
                        with lock:
                            seen[(t, i)] = seen.get((t, i), 0) + 1
                        if not (bits == w).all():
                            errors.append(((t, i), "verdicts"))
                for _ in pending:
                    assert done.acquire(timeout=120)
            except Exception as e:  # noqa: BLE001
                errors.append((t, repr(e)))

        th = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors[:4]
        assert seen == {(t, i): 1 for t in range(16) for i in range(12)}
        assert q.stats()["slow_requests"] == 0 and q.generic_stats()["requests"] > 0


def test_foreign_records_leave_the_sig_cache_alone(engine, oracle, keys, foreign, committee):
    rng = np.random.default_rng(5)
    with engine.queue(ring_records=1024) as q:
        q.generic(True)
        q.sig_cache(1 << 16)
        own = signed(oracle, keys, 40, rng)
        bits = q.wait(q.submit_group(own, np.ones(40, np.uint8)))
        assert (bits == oracle.verify_rec128(own, mode=1)).all()
        s0 = q.sig_stats()
        assert s0["probed"] == 40
        for _ in range(2):
            f = signed(oracle, foreign, 50, rng)
            assert (q.wait(q.submit_group(f, np.ones(50, np.uint8))) == oracle.verify_rec128(f, mode=1)).all()
            mixed = own.copy()
            mixed[::5] = signed(oracle, foreign, 8, rng)  # mixed keys: the whole request is generic, no record probes
            assert (q.wait(q.submit_group(mixed, np.ones(40, np.uint8))) == oracle.verify_rec128(mixed, mode=1)).all()
        assert q.sig_stats() == s0
        assert q.generic_stats()["requests"] == 4


def test_cert_cache_span_with_a_foreign_key_is_inserted_and_hits(engine, oracle, keys, foreign, committee):
    """A Timeout-shaped request whose QC votes include a foreign key verifies on the generic path; its QC span enters the
    certificate cache, and a later copy of the span is a hit."""
    rng = np.random.default_rng(6)
    seeds = np.concatenate([foreign[0][:1], keys[0][:20], foreign[0][1:2]])  # a foreign author too: its record alone is generic
    pks = np.concatenate([foreign[1][:1], keys[1][:20], foreign[1][1:2]])
    pres = [rng.bytes(16), rng.bytes(40)]
    mi = np.array([0] + [1] * 21, np.uint32)
    modes = np.array([0] + [1] * 21, np.uint8)
    r = _sign_with(oracle, seeds, pks, pres, mi, modes, np.arange(22, dtype=np.uint32))
    w = want(oracle, r)
    assert w.all()
    with engine.queue(ring_records=1024) as q:
        q.generic(True)
        q.cert_cache(1 << 20)
        sub = lambda: retry(lambda: q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"]))  # noqa: E731
        assert (q.wait(sub()) == w).all()
        c1, g1 = q.cert_stats(), q.generic_stats()
        assert c1["inserted"] == 1 and g1["requests"] == 1 and g1["records"] == 22
        assert (q.wait(sub()) == w).all()
        c2, g2 = q.cert_stats(), q.generic_stats()
        assert c2["hits"] == c1["hits"] + 1 and c2["records_answered"] == c1["records_answered"] + 21
        assert g2["requests"] == 2 and g2["records"] == 23  # only the author record entered the ring
        assert q.stats()["slow_requests"] == 0


def _sign_with(oracle, seeds, pks, pres, mi, modes, kidx):
    """Records i signed by key kidx[i] over SHA-512(pres[mi[i]])[..32], in the layout of test_queue_msgs.make_req."""
    off = np.zeros(len(pres) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in pres])
    dig = np.array([np.frombuffer(hashlib.sha512(p).digest()[:32], np.uint8) for p in pres])
    sig = oracle.sign_batch(seeds, pks, kidx, dig[mi].reshape(-1), np.arange(len(mi) + 1, dtype=np.uint64) * 32)
    return dict(pre=np.frombuffer(b"".join(pres), np.uint8), off=off, sig=sig, pk=pks[kidx].copy(), mi=mi, modes=modes)


def test_committee_changes_with_generic_requests_in_flight(engine, oracle, keys, foreign, no_committee):
    """register and update while generic requests are in flight: those complete with the oracle's verdicts, and requests submitted
    afterwards are judged against the new committee (a newly registered key takes the device path, a removed one the generic
    path)."""
    rng = np.random.default_rng(7)
    with engine.queue(ring_records=2048) as q:
        q.generic(True)
        burst = [signed(oracle, keys, 64, rng) for _ in range(12)]
        tickets = [q.submit(r, mode=i % 2) for i, r in enumerate(burst)]
        _register(engine, keys[1][:512])
        for i, (t, r) in enumerate(zip(tickets, burst)):
            assert (q.wait(t) == oracle.verify_rec128(r, mode=i % 2)).all()
        s0, g0 = q.stats(), q.generic_stats()
        own = signed(oracle, (keys[0][:512], keys[1][:512]), 30, rng)
        assert (q.wait(q.submit(own, mode=0)) == oracle.verify_rec128(own, mode=0)).all()
        assert q.stats()["small_launches"] == s0["small_launches"] + 1 and q.generic_stats() == g0
        # update: add a foreign key while generic requests are in flight; it then takes the device path
        f = signed(oracle, (foreign[0][:1], foreign[1][:1]), 20, rng)
        tickets = [q.submit(signed(oracle, foreign, 8, rng), mode=1) for _ in range(6)]
        idx = engine.committee_update(add=foreign[1][:1])
        assert len(idx) == 1
        for t in tickets:
            q.wait(t)
        g1 = q.generic_stats()
        assert (q.wait(q.submit(f, mode=0)) == oracle.verify_rec128(f, mode=0)).all()
        assert q.generic_stats() == g1
        assert q.stats()["slow_requests"] == 0
