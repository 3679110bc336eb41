"""The verify queue's signature cache (hs_queue_sig_cache, VerifyQueue.sig_cache): records the queue's kernels accepted are kept in
HBM, so the same record later is a probe that hits instead of a verify.  Every verdict must equal the oracle's and the same request's
on a queue with the cache off; the counters show the probes, hits, inserts and evictions."""
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial
from test_queue_msgs import K, _clear, _register, _sign, want

pytestmark = pytest.mark.gpu
BULK_MIN = 1002
L = 2**252 + 27742317777372353535851937790883648493


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(7900)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture()
def committee(engine, keys):
    _register(engine, keys[1])
    yield
    _clear(engine)


@pytest.fixture()
def queues(engine, committee):
    with engine.queue(ring_records=2048) as q, engine.queue(ring_records=2048) as plain:
        q.sig_cache(1 << 20)  # 262,144 buckets: the exact counts below need no bucket to overflow (the index key is random)
        yield q, plain


def records(oracle, keys, n, rng, corrupt=0.05):
    """n (sig | pk | msg) records over random 32-byte Digests by random committee keys; `corrupt` of them get a flipped bit."""
    seeds, pks = keys
    kidx = rng.integers(0, K, n).astype(np.uint32)
    msgs = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sig = oracle.sign_batch(seeds, pks, kidx, msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    recs = np.concatenate([sig, pks[kidx], msgs], axis=1)
    for i in np.flatnonzero(rng.random(n) < corrupt):
        recs[i, int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
    return recs


def oracle_bits(oracle, recs, modes):
    w = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    return w[np.asarray(modes, np.intp), np.arange(len(recs))]


def submit_group(q, recs, modes):
    while (t := q.submit_group(recs, modes)) is None:
        threading.Event().wait(0.0005)
    return t


def run(q, plain, oracle, recs, modes):
    """One request through the cached queue: its verdicts equal the oracle's and the cache-off queue's.  Returns them and the change
    of the cache's counters."""
    modes = np.broadcast_to(np.asarray(modes, np.uint8), (len(recs),)).copy()
    s0 = q.sig_stats()
    if len(recs) <= 64 and (modes == modes[0]).all():
        bits = q.wait(q.submit(recs, mode=int(modes[0])))
    else:
        bits = q.wait(submit_group(q, recs, modes))
    s1 = q.sig_stats()
    w = oracle_bits(oracle, recs, modes)
    assert (bits == w).all(), np.flatnonzero(bits != w)[:8]
    assert (plain.wait(submit_group(plain, recs, modes)) == bits).all()
    return bits, {k: s1[k] - s0[k] for k in s0 if k != "entries_held"}


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n", [1, 7, 64, 300])
def test_second_pass_hits_in_k_verify_small(engine, oracle, keys, queues, mode, n):
    q, plain = queues
    recs = records(oracle, keys, n, np.random.default_rng(100 + n))
    eq = oracle.verify_rec128(recs, mode=1)
    before = q.stats()
    _, d = run(q, plain, oracle, recs, mode)
    assert d == dict(probed=n, hits=0, inserts=int(eq.sum()), evictions=0)
    _, d = run(q, plain, oracle, recs, mode)
    assert d == dict(probed=n, hits=int(eq.sum()), inserts=0, evictions=0)
    assert q.stats()["bulk_launches"] == before["bulk_launches"]


@pytest.mark.parametrize("mode", [0, 1])
def test_second_pass_hits_in_k_verify_bulk_across_the_ring_end(engine, oracle, keys, queues, mode):
    q, plain = queues
    rng = np.random.default_rng(200 + mode)
    run(q, plain, oracle, records(oracle, keys, 1000, rng), mode)  # the ring's tail at 1,000 of 2,048
    recs = records(oracle, keys, BULK_MIN + 98, rng)
    eq = int(oracle.verify_rec128(recs, mode=1).sum())
    b0 = q.stats()["bulk_launches"]
    _, d = run(q, plain, oracle, recs, mode)  # wraps the ring's end
    assert d == dict(probed=len(recs), hits=0, inserts=eq, evictions=0)
    _, d = run(q, plain, oracle, recs, mode)
    assert d == dict(probed=len(recs), hits=eq, inserts=0, evictions=0)
    assert q.stats()["bulk_launches"] == b0 + 2


def test_batch_eq_only_records_keep_both_verdicts_and_rejected_records_are_never_cached(engine, oracle, keys):
    adv = make_adversarial(oracle, 4000, seed=3)
    eq, st = oracle.verify_rec128(adv, 1), oracle.verify_rec128(adv, 0)
    pks = np.unique(np.concatenate([keys[1], adv[:, 64:96]]), axis=0)
    valid = engine.committee_register(pks)
    try:
        reg = {bytes(k) for k, v in zip(pks, valid) if v}
        on_device = np.array([bytes(r[64:96]) in reg for r in adv])
        small = adv[np.flatnonzero(eq & ~st & on_device)[:64]]
        bad = adv[np.flatnonzero(~eq & on_device)[:64]]
        assert len(small) and len(bad)
        with engine.queue() as q, engine.queue() as plain:
            q.sig_cache(1 << 12)
            bits, d = run(q, plain, oracle, small, 1)
            assert bits.all() and d["inserts"] == len(small)
            bits, d = run(q, plain, oracle, small, 0)  # a hit answers strict from the stored flags
            assert not bits.any() and d["hits"] == len(small)
            bits, d = run(q, plain, oracle, small, 1)
            assert bits.all() and d["hits"] == len(small)
            for mode in (1, 0, 1):
                bits, d = run(q, plain, oracle, bad, mode)
                assert not bits.any() and d == dict(probed=len(bad), hits=0, inserts=0, evictions=0)
    finally:
        _clear(engine)


def test_near_misses_are_verified(engine, oracle, keys, queues):
    q, plain = queues
    base = records(oracle, keys, 8, np.random.default_rng(300), corrupt=0)
    run(q, plain, oracle, base, 1)
    near = []
    for r in base[:2]:
        for byte in (3, 64 + 32 + 5, 40):  # R, M, S
            x = r.copy()
            x[byte] ^= 0x20
            near.append(x)
        x = r.copy()  # another registered key, same (sig, msg)
        x[64:96] = keys[1][(np.flatnonzero((keys[1] == r[64:96]).all(1))[0] + 1) % K]
        near.append(x)
        x = r.copy()  # S + l: the same R, A and M as a cached entry, a non-canonical S
        s = int.from_bytes(x[32:64].tobytes(), "little") + L
        x[32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
        near.append(x)
    near = np.array(near)
    for mode in (0, 1):
        bits, d = run(q, plain, oracle, near, mode)
        assert not bits.any() and d["hits"] == 0 and d["probed"] == len(near)
    _, d = run(q, plain, oracle, base, 0)
    assert d["hits"] == len(base)


def test_a_reused_committee_index_misses(engine, oracle, keys, committee):
    seeds, pks = keys
    order = np.unique(pks, axis=0)  # the committee's indices (see _register)
    rng = np.random.default_rng(400)
    new_seed = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    new_pk = oracle.keygen_batch(new_seed)
    with engine.queue() as q, engine.queue() as plain:
        q.sig_cache(1 << 12)
        recs = records(oracle, keys, 64, rng, corrupt=0)
        run(q, plain, oracle, recs, 1)
        idx = int(np.flatnonzero((order == recs[0, 64:96]).all(1))[0])
        engine.committee_update(add=new_pk, remove=np.array([idx], np.uint32))
        x = recs[:1].copy()
        x[0, 64:96] = new_pk[0]  # K' (maybe at K's old index) with a cached (sig, msg)
        for mode in (1, 0):
            bits, d = run(q, plain, oracle, x, mode)
            assert not bits.any() and d == dict(probed=1, hits=0, inserts=0, evictions=0)
        rest = recs[1:][~(recs[1:, 64:96] == recs[0, 64:96]).all(1)]
        _, d = run(q, plain, oracle, rest, 0)  # no flush: the other records still hit
        assert d["hits"] == len(rest)


def test_view_change_tc_is_answered_from_the_timeouts(engine, oracle, keys, committee):
    """N Timeouts (author strict over round || high_qc round, then the shared high_qc batch-eq) through submit_msgs, then the TC:
    its votes are the Timeouts' author records, so every one of them hits."""
    n = 100
    rng = np.random.default_rng(500)
    qc = _sign(oracle, keys, [rng.bytes(40)], np.zeros(67, np.uint32), np.ones(67, np.uint8), rng)
    authors = rng.permutation(K)[:n]
    tpre = [rng.bytes(16) for _ in range(n)]
    seeds, pks = keys
    from test_queue_cert_cache import _dig
    a_sig = oracle.sign_batch(seeds, pks, authors.astype(np.uint32), np.concatenate([_dig(p) for p in tpre]), np.arange(n + 1, dtype=np.uint64) * 32)
    a_sig[7, 3] ^= 1  # one Timeout with a bad author signature
    with engine.queue(ring_records=16384) as q, engine.queue(ring_records=16384) as plain:
        q.cert_cache(16 << 20)
        q.sig_cache(1 << 14)
        for i in range(n):
            t = dict(pre=np.frombuffer(tpre[i] + qc["pre"].tobytes(), np.uint8), off=np.array([0, 16, 56], np.uint64),
                     sig=np.concatenate([a_sig[i:i + 1], qc["sig"]]), pk=np.concatenate([pks[authors[i:i + 1]], qc["pk"]]),
                     mi=np.array([0] + [1] * 67, np.uint32), modes=np.array([0] + [1] * 67, np.uint8))
            bits = q.wait(q.submit_msgs(t["pre"], t["off"], t["sig"], t["pk"], t["mi"], modes=t["modes"]))
            assert (bits == want(oracle, t)).all()

        def tc(sig, pk, pres):
            return dict(pre=np.frombuffer(b"".join(pres), np.uint8), off=np.arange(len(pres) + 1, dtype=np.uint64) * 16, sig=sig, pk=pk,
                        mi=np.arange(len(pres), dtype=np.uint32), modes=np.zeros(len(pres), np.uint8))

        good = [i for i in range(n) if i != 7][:67]
        cases = [(tc(a_sig[good], pks[authors[good]], [tpre[i] for i in good]), 67, 67)]  # (TC, hits, accepted)
        unseen = _sign(oracle, keys, [rng.bytes(16)], np.zeros(1, np.uint32), np.zeros(1, np.uint8), rng)  # a vote never seen before
        cases.append((tc(np.concatenate([a_sig[good[:66]], unseen["sig"]]), np.concatenate([pks[authors[good[:66]]], unseen["pk"]]),
                         [tpre[i] for i in good[:66]] + [unseen["pre"].tobytes()]), 66, 67))
        bad = a_sig[good].copy()
        bad[10, 50] ^= 4  # a corrupted vote
        cases.append((tc(bad, pks[authors[good]], [tpre[i] for i in good]), 66, 66))
        cases.append((tc(a_sig[[7] + good[:66]], pks[authors[[7] + good[:66]]], [tpre[i] for i in [7] + good[:66]]), 66, 66))  # the bad author
        for r, hits, accepted in cases:
            s0 = q.sig_stats()
            bits = q.wait(q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"]))
            s1 = q.sig_stats()
            w = want(oracle, r)
            assert (bits == w).all() and w.sum() == accepted
            assert (plain.wait(plain.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"])) == bits).all()
            assert s1["probed"] - s0["probed"] == 67 and s1["hits"] - s0["hits"] == hits


def test_eight_threads_on_both_streams_into_a_tiny_table(engine, oracle, keys, committee):
    """Overlapping identical records from 8 threads on both queue streams into 16 buckets: concurrent inserts, probes and evictions
    never change a verdict."""
    rng = np.random.default_rng(600)
    pool = records(oracle, keys, 1500, rng)
    w = np.stack([oracle.verify_rec128(pool, mode=0), oracle.verify_rec128(pool, mode=1)])
    errors = []
    with engine.queue(ring_records=16384) as q:
        q.sig_cache(64)  # 16 buckets
        go = threading.Barrier(8)

        def worker(k):
            r = np.random.default_rng(610 + k)
            go.wait()
            try:
                for it in range(6):
                    if it % 3 == 2:
                        idx = r.choice(len(pool), BULK_MIN + 10, replace=False)
                        modes = r.integers(0, 2, len(idx)).astype(np.uint8)
                        bits = q.wait(submit_group(q, pool[idx], modes))
                    else:
                        idx = r.integers(0, 200, int(r.integers(1, 65)))
                        modes = np.full(len(idx), it % 2, np.uint8)
                        bits = q.wait(q.submit(pool[idx], mode=it % 2))
                    if not (bits == w[modes.astype(np.intp), idx]).all():
                        errors.append((k, it))
            except Exception as ex:  # noqa: BLE001
                errors.append((k, repr(ex)))

        ts = [threading.Thread(target=worker, args=(k,)) for k in range(8)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        s = q.sig_stats()
        assert not errors, errors
        assert s["hits"] > 0 and s["evictions"] > 0 and 0 < s["entries_held"] <= 64


def test_off_by_default_resize_and_teardown_fire_every_callback_once(oracle, keys):
    from hotstuff_b200 import Engine
    rng = np.random.default_rng(700)
    recs = records(oracle, keys, 4 * (BULK_MIN + 20), rng)
    want0 = oracle.verify_rec128(recs, mode=0)
    e = Engine(0)
    try:
        _register(e, keys[1])
        with e.queue() as q:
            q.wait(q.submit(recs[:8]))
            assert q.sig_stats() == dict(probed=0, hits=0, inserts=0, evictions=0, entries_held=0)
        for end in ("resize", "queue", "ctx"):
            q = e.queue(ring_records=16384)
            q.sig_cache(1 << 12)
            fired, lock = {}, threading.Lock()

            def cb(ticket, status, bits):
                with lock:
                    fired.setdefault(ticket, []).append((status, bits))

            expect = {}
            for rep in range(2):
                for i in range(0, len(recs), BULK_MIN + 20):
                    g = recs[i:i + BULK_MIN + 20]
                    expect[q.submit_group(g, callback=cb)] = want0[i:i + BULK_MIN + 20]
                    expect[q.submit(recs[i:i + 5], callback=cb)] = want0[i:i + 5]
                if end == "resize":
                    q.sig_cache(1 << 14 if rep == 0 else 0)  # with launches in flight
            if end == "ctx":
                q.h = None
                e._queues.remove(q)
                e.close()
            else:
                q.close()
            assert sorted(fired) == sorted(expect) and all(len(v) == 1 for v in fired.values())
            for t, v in fired.items():
                assert v[0][0] == 0 and (v[0][1] == expect[t]).all()
    finally:
        e.close()
