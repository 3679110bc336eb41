"""The verify queue's certificate cache (hs_queue_cert_cache, VerifyQueue.cert_cache): a QC that many Timeouts carry is verified once.
Every verdict must equal the oracle's and the same request's on a queue with the cache off; the counters show hits, joins and the
records that entered the ring."""
import hashlib
import threading

import numpy as np
import pytest

from test_queue_msgs import K, _clear, _register, want

pytestmark = pytest.mark.gpu
CACHE = 64 << 20


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(7800)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture()
def committee(engine, keys):
    _register(engine, keys[1])
    yield
    _clear(engine)


def _dig(pre):
    return np.frombuffer(hashlib.sha512(pre).digest()[:32], np.uint8)


def _sign(oracle, keys, kidx, pre):
    seeds, pks = keys
    n = len(kidx)
    sig = oracle.sign_batch(seeds, pks, np.asarray(kidx, np.uint32), np.tile(_dig(pre), n), np.arange(n + 1, dtype=np.uint64) * 32)
    return sig, pks[np.asarray(kidx)].copy()


def make_qc(oracle, keys, votes, rng, bad=()):
    """A QC: `votes` signatures over one 40-byte preimage (hash || round) by distinct keys; the votes in `bad` get a flipped bit."""
    pre = rng.bytes(40)
    sig, pk = _sign(oracle, keys, rng.permutation(K)[:votes] if votes <= K else rng.integers(0, K, votes), pre)
    for i in bad:
        sig[i, 5] ^= 0x10
    return dict(pre=pre, sig=sig, pk=pk)


def timeout(oracle, keys, qc, rng, author_pre_len=16, corrupt=False):
    """A Timeout: one strict author signature over its own preimage, then the high_qc's votes batch-eq over the QC's preimage."""
    a_pre = rng.bytes(author_pre_len)
    a_sig, a_pk = _sign(oracle, keys, [int(rng.integers(0, K))], a_pre)
    if corrupt:
        a_sig[0, 9] ^= 1
    n = 1 + len(qc["sig"])
    return dict(pre=np.frombuffer(a_pre + qc["pre"], np.uint8), off=np.array([0, len(a_pre), len(a_pre) + 40], np.uint64),
                sig=np.concatenate([a_sig, qc["sig"]]), pk=np.concatenate([a_pk, qc["pk"]]),
                mi=(np.arange(n) > 0).astype(np.uint32), modes=(np.arange(n) > 0).astype(np.uint8))


def qc_request(qc):
    """The QC alone as one request (every record is in one span)."""
    n = len(qc["sig"])
    return dict(pre=np.frombuffer(qc["pre"], np.uint8), off=np.array([0, 40], np.uint64), sig=qc["sig"], pk=qc["pk"],
                mi=np.zeros(n, np.uint32), modes=np.ones(n, np.uint8))


def submit(q, r, callback=None):
    while (t := q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"], callback=callback)) is None:
        threading.Event().wait(0.0005)  # no room now: back-pressure
    return t


def delta(a, b):
    return {k: b[k] - a[k] for k in a}


def check(oracle, plain, r, bits):
    """Verdicts equal the oracle's and those of the same request on the queue without the cache."""
    w = want(oracle, r)
    assert len(bits) == len(w) and (bits == w).all(), np.flatnonzero(bits != w)[:8]
    assert (plain.wait(submit(plain, r)) == bits).all()


@pytest.fixture()
def queues(engine, committee):
    with engine.queue(ring_records=16384) as q, engine.queue(ring_records=16384) as plain:
        q.cert_cache(CACHE)
        yield q, plain


def test_hits_after_a_verified_block(engine, oracle, keys, queues):
    """A Block's QC verifies first; every Timeout carrying it is then answered from the cache and puts only its author in the ring."""
    q, plain = queues
    rng = np.random.default_rng(1)
    qc = make_qc(oracle, keys, 669, rng)
    block = timeout(oracle, keys, qc, rng, author_pre_len=136)  # same shape: author strict + the QC's votes
    c0 = q.cert_stats()
    check(oracle, plain, block, q.wait(submit(q, block)))
    c1 = q.cert_stats()
    assert delta(c0, c1) == dict(lookups=1, hits=0, joins=0, records_answered=0, inserted=1, bytes_held=9 + 40 + 96 * 669)
    for k in range(6):
        t = timeout(oracle, keys, qc, rng, corrupt=k == 3)
        s0, c0 = q.stats(), q.cert_stats()
        bits = q.wait(submit(q, t))
        s1, c1 = q.stats(), q.cert_stats()
        assert s1["small_records"] - s0["small_records"] == 1 and s1["bulk_records"] == s0["bulk_records"]
        assert delta(c0, c1) == dict(lookups=1, hits=1, joins=0, records_answered=669, inserted=0, bytes_held=0)
        assert bits[1:].all() and bits[0] == (k != 3)
        check(oracle, plain, t, bits)


def test_eight_threads_submitting_identical_timeouts_join(engine, oracle, keys, queues):
    """8 threads submit Timeouts with the same 1,335-vote QC at once: one verifies it, the others join it (or hit once it is done).
    The threads' submits are serialised by the binding and the GIL, and take about as long as the QC's GPU pass, so the QC is held in
    flight: as the threads are released, records signed by keys outside the committee are submitted first, and the queue's thread
    verifies them on its slow path (about a millisecond each) before it can see the QC's pass complete."""
    q, plain = queues
    rng = np.random.default_rng(2)
    qc = make_qc(oracle, keys, 1335, rng)
    ts = [timeout(oracle, keys, qc, rng, corrupt=i == 5) for i in range(8)]
    f_seeds = rng.integers(0, 256, size=(4, 32), dtype=np.uint8)
    f_pks, f_dig = oracle.keygen_batch(f_seeds), np.frombuffer(rng.bytes(4 * 32), np.uint8).reshape(4, 32)
    f_sig = oracle.sign_batch(f_seeds, f_pks, np.arange(4, dtype=np.uint32), f_dig.reshape(-1), np.arange(5, dtype=np.uint64) * 32)
    slow = np.concatenate([f_sig, f_pks, f_dig], axis=1)
    held = []
    go = threading.Barrier(8, action=lambda: held.extend(q.submit(slow[i:i + 1]) for i in range(4)))
    out = [None] * 8

    def run(i):
        go.wait()
        out[i] = q.wait(submit(q, ts[i]))

    c0, s0 = q.cert_stats(), q.stats()
    th = [threading.Thread(target=run, args=(i,)) for i in range(8)]
    [t.start() for t in th]
    [t.join() for t in th]
    d = delta(c0, q.cert_stats())
    assert d["lookups"] == 8 and d["inserted"] == 1 and d["hits"] + d["joins"] == 7 and d["joins"] >= 1, d
    assert d["records_answered"] == 7 * 1335
    assert [bool(q.wait(t)[0]) for t in held] == list(oracle.verify_rec128(slow, mode=0)) and delta(s0, q.stats())["slow_requests"] == 4
    for t, bits in zip(ts, out):
        check(oracle, plain, t, bits)
    # the same from one thread without waiting in between: every later copy finds the QC in flight or verified
    qc2 = make_qc(oracle, keys, 1335, rng)
    ts2 = [timeout(oracle, keys, qc2, rng) for _ in range(8)]
    c0 = q.cert_stats()
    tickets = [submit(q, t) for t in ts2]
    outs = [q.wait(t) for t in tickets]
    d = delta(c0, q.cert_stats())
    assert d["lookups"] == 8 and d["inserted"] == 1 and d["hits"] + d["joins"] == 7
    for t, bits in zip(ts2, outs):
        check(oracle, plain, t, bits)


def test_misses_on_reordered_votes_another_vote_set_and_a_flipped_bit(engine, oracle, keys, queues):
    q, plain = queues
    rng = np.random.default_rng(3)
    qc = make_qc(oracle, keys, 67, rng)
    check(oracle, plain, t := timeout(oracle, keys, qc, rng), q.wait(submit(q, t)))
    perm = np.roll(np.arange(67), 1)
    reordered = dict(qc, sig=qc["sig"][perm], pk=qc["pk"][perm])
    extra_sig, extra_pk = _sign(oracle, keys, [int(k) for k in rng.integers(0, K, 1)], qc["pre"])
    other_set = dict(qc, sig=np.concatenate([qc["sig"][:-1], extra_sig]), pk=np.concatenate([qc["pk"][:-1], extra_pk]))
    flipped = dict(qc, sig=qc["sig"].copy())
    flipped["sig"][40, 63] ^= 0x01
    for variant, inserts in ((reordered, 1), (other_set, 1), (flipped, 0)):
        t = timeout(oracle, keys, variant, rng)
        c0 = q.cert_stats()
        bits = q.wait(submit(q, t))
        d = delta(c0, q.cert_stats())
        assert d["lookups"] == 1 and d["hits"] == 0 and d["joins"] == 0 and d["inserted"] == inserts, d
        check(oracle, plain, t, bits)
    # the original still hits
    c0 = q.cert_stats()
    check(oracle, plain, t := timeout(oracle, keys, qc, rng), q.wait(submit(q, t)))
    assert delta(c0, q.cert_stats())["hits"] == 1


def test_a_failing_qc_gives_its_joiners_the_failing_bits_and_is_never_inserted(engine, oracle, keys, queues):
    q, plain = queues
    rng = np.random.default_rng(4)
    qc = make_qc(oracle, keys, 1335, rng, bad=(17,))
    ts = [timeout(oracle, keys, qc, rng) for _ in range(8)]
    c0 = q.cert_stats()
    tickets = [submit(q, t) for t in ts]
    outs = [q.wait(t) for t in tickets]
    d = delta(c0, q.cert_stats())
    assert d["lookups"] == 8 and d["inserted"] == 0 and d["hits"] == 0 and d["joins"] <= 7 and d["bytes_held"] == 0, d
    for t, bits in zip(ts, outs):
        assert not bits[1 + 17] and bits[1:].sum() == 1334
        check(oracle, plain, t, bits)
    c0 = q.cert_stats()
    check(oracle, plain, t := timeout(oracle, keys, qc, rng), q.wait(submit(q, t)))
    assert delta(c0, q.cert_stats())["hits"] == 0


def test_lru_eviction_at_a_small_max_bytes(engine, oracle, keys, committee):
    rng = np.random.default_rng(5)
    key = 9 + 40 + 96 * 20
    qcs = [make_qc(oracle, keys, 20, rng) for _ in range(3)]
    with engine.queue() as q, engine.queue() as plain:
        q.cert_cache(2 * key + 100)  # room for two QCs

        def run(i):
            t = timeout(oracle, keys, qcs[i], rng)
            c0 = q.cert_stats()
            check(oracle, plain, t, q.wait(submit(q, t)))
            return delta(c0, q.cert_stats())

        assert run(0)["inserted"] == 1 and run(1)["inserted"] == 1
        assert q.cert_stats()["bytes_held"] == 2 * key
        assert run(0)["hits"] == 1          # QC 0 is now the most recently used
        assert run(2)["inserted"] == 1      # evicts QC 1
        assert q.cert_stats()["bytes_held"] == 2 * key
        assert run(0)["hits"] == 1 and run(2)["hits"] == 1
        d = run(1)
        assert d["hits"] == 0 and d["inserted"] == 1
        q.cert_cache(0)                     # off: everything goes
        assert q.cert_stats()["bytes_held"] == 0
        d = run(1)
        assert d["lookups"] == 0 and d["inserted"] == 0


def test_a_request_answered_entirely_from_the_cache(engine, oracle, keys, queues):
    """The QC alone after it verified: no record enters the ring, yet the ticket completes through wait, poll and a callback that
    runs exactly once on the queue's thread."""
    q, plain = queues
    rng = np.random.default_rng(6)
    qc = make_qc(oracle, keys, 40, rng)
    r = qc_request(qc)
    check(oracle, plain, r, q.wait(submit(q, r)))
    s0, l0 = q.stats(), engine.kernel_launches
    assert q.wait(submit(q, r)).all()
    t = submit(q, r)
    while (bits := q.poll(t)) is None:
        threading.Event().wait(0.0002)
    assert bits.all()
    seen, threads, done = [], [], threading.Event()

    def cb(ticket, status, bools):
        seen.append((ticket, status, bools.copy()))
        threads.append(threading.get_ident())
        done.set()

    t = submit(q, r, callback=cb)
    assert done.wait(10)
    threading.Event().wait(0.05)
    assert len(seen) == 1 and seen[0][0] == t and seen[0][1] == 0 and seen[0][2].all()
    assert threads[0] != threading.get_ident()
    assert q.stats() == s0 and engine.kernel_launches == l0  # nothing launched
    assert q.cert_stats()["hits"] == 3
    # the same thread runs the callback of a request that did launch
    done.clear()
    submit(q, timeout(oracle, keys, make_qc(oracle, keys, 40, rng), rng), callback=cb)
    assert done.wait(10)
    threading.Event().wait(0.05)
    assert len(threads) == 2 and threads[1] == threads[0]


def test_ring_and_arena_limits_count_only_records_that_enter(engine, oracle, keys, committee):
    rng = np.random.default_rng(7)
    # ring: a QC of 4,096 votes fills a 4,096-record ring on its own; a Timeout carrying it has 4,097 records
    qc = make_qc(oracle, keys, 4096, rng)
    t = timeout(oracle, keys, qc, rng)
    with engine.queue(ring_records=4096) as q, engine.queue(ring_records=16384) as plain:
        with pytest.raises(RuntimeError):
            q.submit_msgs(t["pre"], t["off"], t["sig"], t["pk"], t["mi"], modes=t["modes"])  # HS_ERR_ARG: more than the ring
        q.cert_cache(CACHE)
        check(oracle, plain, r := qc_request(qc), q.wait(submit(q, r)))
        s0 = q.stats()
        bits = q.wait(submit(q, t))
        assert q.stats()["small_records"] - s0["small_records"] == 1
        check(oracle, plain, t, bits)
    # arena: 64 records hold 4,096 preimage-arena bytes; a 3,000-byte QC preimage fits alone, with a 2,000-byte author preimage not
    big = dict(pre=rng.bytes(3000))
    big["sig"], big["pk"] = _sign(oracle, keys, rng.permutation(K)[:20], big["pre"])
    a_pre = rng.bytes(2000)
    a_sig, a_pk = _sign(oracle, keys, [3], a_pre)
    t = dict(pre=np.frombuffer(a_pre + big["pre"], np.uint8), off=np.array([0, 2000, 5000], np.uint64), sig=np.concatenate([a_sig, big["sig"]]),
             pk=np.concatenate([a_pk, big["pk"]]), mi=(np.arange(21) > 0).astype(np.uint32), modes=(np.arange(21) > 0).astype(np.uint8))
    r = dict(pre=np.frombuffer(big["pre"], np.uint8), off=np.array([0, 3000], np.uint64), sig=big["sig"], pk=big["pk"],
             mi=np.zeros(20, np.uint32), modes=np.ones(20, np.uint8))
    with engine.queue(ring_records=64) as q, engine.queue(ring_records=16384) as plain:
        with pytest.raises(RuntimeError):
            q.submit_msgs(t["pre"], t["off"], t["sig"], t["pk"], t["mi"], modes=t["modes"])  # HS_ERR_ARG: more than the arena
        q.cert_cache(CACHE)
        check(oracle, plain, r, q.wait(submit(q, r)))
        d0 = q.digest_stats()
        bits = q.wait(submit(q, t))
        assert q.digest_stats()["preimage_bytes"] - d0["preimage_bytes"] == 2000
        check(oracle, plain, t, bits)


def test_submit_group_spans(engine, oracle, keys, queues):
    """Digest spans of submit_group hit each other, never a preimage span of submit_msgs with the same votes."""
    q, plain = queues
    rng = np.random.default_rng(8)
    qc = make_qc(oracle, keys, 100, rng)

    def recs(t):
        pre, off = t["pre"].tobytes(), t["off"]
        dig = np.array([_dig(pre[int(off[j]):int(off[j + 1])]) for j in range(len(off) - 1)])
        out = np.zeros((len(t["mi"]), 128), np.uint8)
        out[:, :64], out[:, 64:96], out[:, 96:] = t["sig"], t["pk"], dig[t["mi"]]
        return out

    for k in range(3):
        t = timeout(oracle, keys, qc, rng, corrupt=k == 1)
        c0 = q.cert_stats()
        rr = recs(t)
        bits = q.wait(q.submit_group(rr, modes=t["modes"]))
        d = delta(c0, q.cert_stats())
        assert d["lookups"] == 1 and d["hits"] == int(k > 0) and d["inserted"] == int(k == 0), d
        assert (bits == want(oracle, t)).all() and (plain.wait(plain.submit_group(rr, modes=t["modes"])) == bits).all()
    c0 = q.cert_stats()
    check(oracle, plain, t := timeout(oracle, keys, qc, rng), q.wait(submit(q, t)))
    d = delta(c0, q.cert_stats())
    assert d["hits"] == 0 and d["inserted"] == 1


def test_committee_update_with_the_cache_warm(engine, oracle, keys, queues):
    q, plain = queues
    rng = np.random.default_rng(9)
    qc = make_qc(oracle, keys, 200, rng)
    check(oracle, plain, t := timeout(oracle, keys, qc, rng), q.wait(submit(q, t)))
    uniq = np.unique(keys[1], axis=0)  # the registered committee, in index order
    gone = qc["pk"][:5]
    engine.committee_update(remove=[int(np.flatnonzero((uniq == p).all(axis=1))[0]) for p in gone])
    try:
        for k in range(3):
            c0 = q.cert_stats()
            check(oracle, plain, t := timeout(oracle, keys, qc, rng, corrupt=k == 2), q.wait(submit(q, t)))
            assert delta(c0, q.cert_stats())["hits"] == 1
    finally:
        engine.committee_update(add=gone)


@pytest.mark.parametrize("how", ["queue", "context"])
def test_teardown_with_joiners_pending(oracle, keys, how):
    """Destroying the queue (or its context) with a primary in flight and joiners waiting completes every request: each callback
    fires exactly once, with the verdicts."""
    from hotstuff_b200 import Engine
    rng = np.random.default_rng(10)
    e = Engine(0)
    try:
        _register(e, keys[1])
        q = e.queue(ring_records=16384)
        q.cert_cache(CACHE)
        qc = make_qc(oracle, keys, 1335, rng)
        ts = [timeout(oracle, keys, qc, rng, corrupt=i == 2) for i in range(12)]
        got = {}
        lock = threading.Lock()

        def cb(i):
            def f(ticket, status, bools):
                with lock:
                    got.setdefault(i, []).append((status, bools.copy()))
            return f

        for i, t in enumerate(ts):
            submit(q, t, callback=cb(i))
        if how == "queue":
            q.close()
        else:  # hs_ctx_destroy tears down the queue still attached to it
            q.h = None
            e._queues.remove(q)
            e.close()
        assert sorted(got) == list(range(12)) and all(len(v) == 1 for v in got.values())
        for i, t in enumerate(ts):
            status, bits = got[i][0]
            assert status == 0 and (bits == want(oracle, t)).all()
    finally:
        e.close()
