"""Preimage requests through the verify queue (hs_queue_submit_msgs, VerifyQueue.submit_msgs): one consensus message's signatures with
the signed preimages instead of their Digests, hashed on the GPU by k_queue_digests.  Record i's verdict must equal the oracle on
(sig[i], pk[i], SHA-512(preimage_{msg_idx[i]})[..32]) in modes[i], and item i of hs_verify_groups on the same arrays as one group."""
import hashlib
import os
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial, make_workload, to_rec128

pytestmark = pytest.mark.gpu
BULK_MIN = 1002
K = 1024  # committee keys


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(7700)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


def _register(engine, pks):
    engine.committee_register(np.unique(np.asarray(pks, np.uint8).reshape(-1, 32), axis=0))


def _clear(engine):
    engine.committee_register(np.zeros((0, 32), np.uint8))


def make_req(oracle, keys, shape, n, rng, pre_len=136, corrupt=0.02, key_lo=0, key_hi=K):
    """A request of n records in the shape of one consensus message:
      vote     : every record over one 40-byte preimage, strict
      timeout  : author strict over a 16-byte preimage, then the high_qc's votes batch-eq over a 40-byte preimage
      tc       : record i strict over its own 16-byte preimage (tc.round || high_qc_round)
      block_tc : author strict over the Block preimage (pre_len bytes), QC votes batch-eq over 40 bytes, TC votes strict over 16
    Every shape but `tc` also carries one preimage that no record names.  `corrupt` of the signatures get a flipped bit."""
    seeds, pks = keys
    if shape == "vote":
        pres, mi, modes = [rng.bytes(40), rng.bytes(8)], np.zeros(n, np.uint32), np.zeros(n, np.uint8)
    elif shape == "timeout":
        pres = [rng.bytes(16), rng.bytes(3), rng.bytes(40)]
        mi = np.full(n, 2, np.uint32)
        mi[0] = 0
        modes = np.ones(n, np.uint8)
        modes[0] = 0
    elif shape == "tc":
        pres, mi, modes = [rng.bytes(16) for _ in range(n)], np.arange(n, dtype=np.uint32), np.zeros(n, np.uint8)
    elif shape == "block_tc":
        q = min(n - 1, (2 * n) // 3)
        t = n - 1 - q
        pres = [rng.bytes(pre_len), rng.bytes(40), rng.bytes(77)] + [rng.bytes(16) for _ in range(t)]
        mi = np.concatenate([[0], np.ones(q), 3 + np.arange(t)]).astype(np.uint32)
        modes = np.concatenate([[0], np.ones(q), np.zeros(t)]).astype(np.uint8)
    else:
        raise ValueError(shape)
    return _sign(oracle, keys, pres, mi, modes, rng, corrupt, key_lo, key_hi)


def _sign(oracle, keys, pres, mi, modes, rng, corrupt=0.0, key_lo=0, key_hi=K):
    seeds, pks = keys
    n = len(mi)
    off = np.zeros(len(pres) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in pres])
    dig = np.array([np.frombuffer(hashlib.sha512(p).digest()[:32], np.uint8) for p in pres]).reshape(-1, 32)
    kidx = rng.integers(key_lo, key_hi, n).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, kidx, dig[mi].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    for i in np.flatnonzero(rng.random(n) < corrupt):
        sig[i, int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
    pre = np.frombuffer(b"".join(pres), np.uint8) if off[-1] else np.zeros(0, np.uint8)
    return dict(pre=pre, off=off, sig=sig, pk=pks[kidx].copy(), mi=np.asarray(mi, np.uint32), modes=np.asarray(modes, np.uint8))


def want(oracle, r):
    """The oracle's verdict of each record over SHA-512(its preimage)[..32] (hashlib), in its mode."""
    pre, off = r["pre"].tobytes(), r["off"]
    dig = np.array([np.frombuffer(hashlib.sha512(pre[int(off[j]):int(off[j + 1])]).digest()[:32], np.uint8) for j in range(len(off) - 1)])
    recs = np.zeros((len(r["mi"]), 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = r["sig"], r["pk"], dig[r["mi"]]
    return np.where(r["modes"] == 1, oracle.verify_rec128(recs, mode=1), oracle.verify_rec128(recs, mode=0))


def groups_items(engine, r):
    n = len(r["mi"])
    g, items = engine.verify_groups(r["pre"], r["off"], r["sig"], r["mi"], np.zeros(n, np.uint32), 1, mode=r["modes"], pk=r["pk"], want_items=True)
    assert g[0] == items.all()
    return items


def submit(q, r, callback=None):
    while (t := q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"], callback=callback)) is None:
        threading.Event().wait(0.0005)  # no room now: back-pressure
    return t


def check(engine, oracle, r, bits):
    w = want(oracle, r)
    assert len(bits) == len(w) and (bits == w).all(), np.flatnonzero(bits != w)[:8]
    assert (bits == groups_items(engine, r)).all()


def distinct(r):
    return len(np.unique(r["mi"]))


def test_shapes_on_the_device_path_cost_two_launches(engine, oracle, keys):
    """Vote-, Timeout-, TC- and Block-with-TC-shaped requests of 1, 64, 65 and 668 records, then BULK_MIN - 1, BULK_MIN and 6,668 records
    on a 16,384-record ring, each alone: verdicts equal the oracle and hs_verify_groups, the request costs exactly k_queue_digests plus
    one verify launch on the expected kernel, and each distinct named preimage is hashed once."""
    rng = np.random.default_rng(1)
    _register(engine, keys[1])
    try:
        with engine.queue(ring_records=16384) as q:
            cases = [(s, n) for s in ("vote", "timeout", "tc", "block_tc") for n in (1, 64, 65, 668)]
            cases += [("block_tc", BULK_MIN - 1), ("tc", BULK_MIN), ("block_tc", 6668)]
            for shape, n in cases:
                r = make_req(oracle, keys, shape, n, rng)
                s0, d0, l0 = q.stats(), q.digest_stats(), engine.kernel_launches
                bits = q.wait(submit(q, r))
                s1, d1 = q.stats(), q.digest_stats()
                assert engine.kernel_launches - l0 == 2, (shape, n)
                bulk = n >= BULK_MIN
                assert s1["bulk_launches"] - s0["bulk_launches"] == int(bulk) and s1["small_launches"] - s0["small_launches"] == int(not bulk)
                assert s1["slow_requests"] == s0["slow_requests"]
                assert d1["digest_launches"] - d0["digest_launches"] == 1 and d1["msgs_requests"] - d0["msgs_requests"] == 1
                assert d1["preimages"] - d0["preimages"] == distinct(r), (shape, n)
                named = sorted(set(int(j) for j in r["mi"]))
                assert d1["preimage_bytes"] - d0["preimage_bytes"] == sum(int(r["off"][j + 1] - r["off"][j]) for j in named)
                check(engine, oracle, r, bits)
    finally:
        _clear(engine)


def test_preimage_lengths_and_a_flipped_preimage_byte(engine, oracle, keys):
    """Preimages of 0, 1, 16, 40, 111, 112, 127, 128, 239, 240 bytes and a multi-KB Block preimage, three honest records each: every one
    accepts, so every Digest the kernel wrote is right.  Then one byte of one preimage flipped after signing: exactly its records reject."""
    rng = np.random.default_rng(2)
    lens = [0, 1, 16, 40, 111, 112, 127, 128, 239, 240, 6000]
    pres = [rng.bytes(L) for L in lens]
    mi = np.repeat(np.arange(len(lens)), 3).astype(np.uint32)
    modes = (np.arange(len(mi)) % 2).astype(np.uint8)
    r = _sign(oracle, keys, pres, mi, modes, rng)
    _register(engine, keys[1])
    try:
        with engine.queue() as q:
            bits = q.wait(submit(q, r))
            assert bits.all()
            check(engine, oracle, r, bits)
            for j in (3, 8, 10):                                 # 40, 239 bytes and the multi-KB preimage
                bad = dict(r, pre=r["pre"].copy())
                bad["pre"][int(r["off"][j]) + len(pres[j]) // 2] ^= 0x01
                bits = q.wait(submit(q, bad))
                assert (bits == (mi != j)).all()
                check(engine, oracle, bad, bits)
    finally:
        _clear(engine)


def test_golden_adversarial_and_corrupted_records(engine, oracle, golden, keys):
    """Golden and adversarial (sig, pk) pairs (torsion, non-canonical S, small-order and undecodable points) and corrupted honest records
    over GPU-hashed preimages, on the device path (every key registered) and on the slow path (no committee)."""
    rng = np.random.default_rng(3)
    vs = [v for v in golden["vectors"] if len(v["msg"]) == 64]
    gold = np.array([np.frombuffer(bytes.fromhex(v["sig"] + v["pk"]), np.uint8) for v in vs])
    adv = make_adversarial(oracle, 400, seed=3)
    r = make_req(oracle, keys, "block_tc", 668, rng, corrupt=0.1)
    odd = np.concatenate([gold, adv[:, :96]])[:500]
    sel = rng.choice(np.arange(1, 668), len(odd), replace=False)  # over the QC preimage (batch-eq) and the TC preimages (strict)
    r["sig"][sel], r["pk"][sel] = odd[:, :64], odd[:, 64:96]
    _register(engine, r["pk"])
    try:
        with engine.queue() as q:
            check(engine, oracle, r, q.wait(submit(q, r)))
    finally:
        _clear(engine)
    with engine.queue() as q:
        s0 = q.stats()
        check(engine, oracle, r, q.wait(submit(q, r)))
        assert q.stats()["slow_requests"] - s0["slow_requests"] == 1


def test_eight_threads_mix_submit_group_and_msgs(engine, oracle, keys):
    """8 threads interleave submit, submit_group and submit_msgs, consumed by wait, poll and callback in turn.  Results are checked only
    after every callback has fired; callback statuses are asserted here, not inside the callback."""
    rng = np.random.default_rng(5)
    reqs = [make_req(oracle, keys, s, n, rng) for s, n in [("vote", 3), ("timeout", 40), ("tc", 65), ("block_tc", 300), ("tc", 7), ("block_tc", 90)]]
    wants = [want(oracle, r) for r in reqs]
    recs = to_rec128(make_workload(oracle, 512, n_keys=64, seed=6, corrupt_frac=0.05))
    rw = np.stack([oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)])
    _register(engine, np.concatenate([keys[1], recs[:, 64:96]]))
    out, errors, cv, pending = [], [], threading.Condition(), [0]

    def worker(t):
        trng = np.random.default_rng(50 + t)
        held = []
        try:
            for k in range(12):
                how, kind = (k + t) % 3, (k + 2 * t) % 3
                cb = None
                if how == 2:
                    def cb(ticket, status, bits, key=(t, k)):
                        with cv:
                            out.append((key, status, bits))
                            pending[0] -= 1
                            cv.notify_all()
                    with cv:
                        pending[0] += 1
                if kind == 0:
                    j = int(trng.integers(0, len(reqs)))
                    ticket, expect = submit(q, reqs[j], cb), wants[j]
                else:
                    idx = trng.integers(0, len(recs), 5 if kind == 1 else 120)
                    modes = trng.integers(0, 2, len(idx)).astype(np.uint8)
                    if kind == 1:
                        modes[:] = modes[0]
                        while (ticket := q.submit(recs[idx], mode=int(modes[0]), callback=cb)) is None:
                            threading.Event().wait(0.0005)
                    else:
                        while (ticket := q.submit_group(recs[idx], modes, callback=cb)) is None:
                            threading.Event().wait(0.0005)
                    expect = rw[modes.astype(np.intp), idx]
                expects[(t, k)] = expect
                held.append((ticket, how, (t, k)))
            for ticket, how, key in held:
                if how == 0:
                    bits = q.wait(ticket)
                elif how == 1:
                    while (bits := q.poll(ticket)) is None:
                        pass
                else:
                    continue
                with cv:
                    out.append((key, 0, bits))
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))

    expects = {}
    try:
        with engine.queue(ring_records=2048) as q:
            ts = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
            for t in ts:
                t.start()
            for t in ts:
                t.join()
            assert not errors, errors[:3]
            with cv:
                assert cv.wait_for(lambda: pending[0] == 0, timeout=300), "%d callbacks never fired" % pending[0]
        assert len(out) == 8 * 12
        for key, status, bits in out:
            assert status == 0 and (bits == expects[key]).all(), key
    finally:
        _clear(engine)


def test_ring_and_arena_wrap(engine, oracle, keys):
    """300-record TC requests one after the other on a 1,024-record ring (a 64 KB arena, 8,416 bytes a request): requests straddle the
    ring's end, and the arena's end is crossed (the request that would straddle it starts over at its beginning)."""
    rng = np.random.default_rng(8)
    _register(engine, keys[1])
    try:
        with engine.queue(ring_records=1024) as q:
            for k in range(14):                                 # 4,200 records: the ring wraps 4 times, the arena at least once
                r = make_req(oracle, keys, "tc" if k % 2 else "block_tc", 300, rng, pre_len=1000 + 97 * k)
                check(engine, oracle, r, q.wait(submit(q, r)))
    finally:
        _clear(engine)


def test_arena_back_pressure_and_argument_errors(engine, oracle, keys):
    """On a 1,024-record ring (a 64 KB arena), a request over one 40 KB preimage leaves no arena room for a second while the ring still
    has plenty: the second is refused (None) and accepted once the first has completed.  Bad arguments are HS_ERR_ARG."""
    from hotstuff_b200 import EngineError
    rng = np.random.default_rng(9)
    big = _sign(oracle, keys, [rng.bytes(40000)], np.zeros(8, np.uint32), np.zeros(8, np.uint8), rng)
    _register(engine, keys[1])
    try:
        with engine.queue(ring_records=1024) as q:
            for _ in range(3):
                t = q.submit_msgs(big["pre"], big["off"], big["sig"], big["pk"], big["mi"])
                assert t is not None
                assert q.submit_msgs(big["pre"], big["off"], big["sig"], big["pk"], big["mi"]) is None   # 16 of 1,024 ring records
                assert q.wait(t).all()
                t = q.submit_msgs(big["pre"], big["off"], big["sig"], big["pk"], big["mi"])
                assert t is not None and q.wait(t).all()
            r = make_req(oracle, keys, "block_tc", 30, rng)

            def bad(**kw):
                a = dict(preimages=r["pre"], pre_off=r["off"], sig=r["sig"], pk=r["pk"], msg_idx=r["mi"], modes=r["modes"])
                a.update(kw)
                with pytest.raises(EngineError, match="status 2"):
                    q.submit_msgs(**a)

            bad(sig=r["sig"][:0], pk=r["pk"][:0], msg_idx=r["mi"][:0], modes=r["modes"][:0])          # n = 0
            off = r["off"].copy()
            off[2], off[3] = off[3], off[2]
            bad(pre_off=off)                                                                           # non-monotone
            mi = r["mi"].copy()
            mi[4] = len(r["off"]) - 1
            bad(msg_idx=mi)                                                                            # msg_idx >= n_msgs
            modes = r["modes"].copy()
            modes[5] = 2
            bad(modes=modes)                                                                           # mode byte > 1
            huge = np.zeros(70000, np.uint8)
            bad(preimages=huge, pre_off=np.array([0, 70000], np.uint64), msg_idx=np.zeros(30, np.uint32))   # more than the arena
            check(engine, oracle, r, q.wait(submit(q, r)))                                              # the queue still works
    finally:
        _clear(engine)


def test_slow_path_and_split_dispatch(engine, oracle, keys):
    """An unregistered key sends a request to the slow path (one hs_verify_groups call): parity, and it shows in the slow-path
    counters.  A 300-record slow request between device requests never rides in a launch: the small kernel carries exactly the device
    requests' records, whatever the grouping of the dispatches."""
    rng = np.random.default_rng(10)
    _clear(engine)
    with engine.queue() as q:
        r = make_req(oracle, keys, "block_tc", 200, rng)
        s0, d0 = q.stats(), q.digest_stats()
        check(engine, oracle, r, q.wait(submit(q, r)))
        s1, d1 = q.stats(), q.digest_stats()
        assert s1["slow_requests"] - s0["slow_requests"] == 1 and s1["slow_records"] - s0["slow_records"] == 200
        assert d1["digest_launches"] == d0["digest_launches"] and d1["msgs_requests"] - d0["msgs_requests"] == 1
    engine.committee_register(keys[1][1:])                       # key 0 unregistered
    try:
        with engine.queue(ring_records=16384) as q:
            for _ in range(3):
                dev = [make_req(oracle, keys, s, n, rng, key_lo=1) for s, n in (("tc", 300), ("block_tc", 300), ("timeout", 64))]
                slow = make_req(oracle, keys, "block_tc", 300, rng)
                slow["pk"][7] = keys[1][0]
                small = make_req(oracle, keys, "tc", 20, rng)
                small["pk"][3] = keys[1][0]                      # a slow-path rider of 20 records
                order = [dev[0], slow, dev[1], small, dev[2]]
                s0 = q.stats()
                tickets = [submit(q, r) for r in order]
                for t, r in zip(tickets, order):
                    check(engine, oracle, r, q.wait(t))
                s1 = q.stats()
                assert s1["slow_requests"] - s0["slow_requests"] == 2
                carried = s1["small_records"] - s0["small_records"]
                assert carried in (664, 684), carried           # the device records, plus the 20-record rider when it rode along
    finally:
        _clear(engine)


def test_msgs_across_committee_update(engine, oracle, keys):
    """hs_committee_update with preimage requests in flight: they complete correctly; a request signed by a new validator afterwards takes
    the device path (two launches)."""
    rng = np.random.default_rng(11)
    engine.committee_register(keys[1][:512])
    try:
        with engine.queue() as q:
            reqs = [make_req(oracle, keys, s, 200, rng, key_hi=512) for s in ("tc", "block_tc") * 5]
            tickets = [submit(q, r) for r in reqs]
            engine.committee_update(add=keys[1][512:520], remove=np.arange(4, dtype=np.uint32))
            for t, r in zip(tickets, reqs):
                check(engine, oracle, r, q.wait(t))
            r = make_req(oracle, keys, "block_tc", 100, rng, key_lo=512, key_hi=520, corrupt=0.0)
            l0 = engine.kernel_launches
            assert q.wait(submit(q, r)).all()
            assert engine.kernel_launches - l0 == 2
    finally:
        _clear(engine)


def _threads():
    return len(os.listdir("/proc/self/task"))


def test_msgs_teardown_fires_every_callback_once(oracle, keys):
    """hs_queue_destroy and hs_ctx_destroy with preimage requests in flight, half on the device path and half holding key 0 (unregistered,
    slow path): every callback fires once with the right verdicts and no thread is left."""
    from hotstuff_b200 import Engine
    rng = np.random.default_rng(12)
    e = Engine(0)
    try:
        e.committee_register(keys[1][1:])
        e.queue().close()
        for via_ctx in (False, True):
            before = _threads()
            q = e.queue(ring_records=8192)
            fired, lock = {}, threading.Lock()

            def cb(ticket, status, bits):
                with lock:
                    fired.setdefault(ticket, []).append((status, bits))

            expect = {}
            for k in range(8):
                r = make_req(oracle, keys, ("tc", "block_tc")[k % 2], 256, rng, key_lo=1)
                if k % 4 == 0:
                    r["pk"][5] = keys[1][0]
                expect[q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"], callback=cb)] = want(oracle, r)
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


def test_receiver_path_ingest_one_frame_then_submit_msgs(engine, oracle, golden):
    """Frames from the reference's fixtures go one at a time through hs_ingest_consensus_frames and submit_msgs; each frame's AND over its
    verdicts equals its group bit from hs_verify_groups on the ingest of all frames.  A SyncRequest and a malformed frame are not
    submitted."""
    import bincode_ref as bc
    import messages_scenarios as sc
    from hotstuff_b200 import crypto, messages, wire
    fx = sc.Fixtures(oracle, golden, engine)
    chain = fx.chain(4)
    blk_tc = fx.block(1, 9, qc=chain[3].qc, tc=fx.tc(8), payload=[fx.d(b"p%d" % i) for i in range(40)])
    v = messages.Vote(fx.d(chain[0].preimage()), 1, fx.pks[3], crypto.Signature())
    v.signature = fx.sign(3, fx.d(messages.vote_preimage(v.hash, v.round)))
    bad_sig = fx.block(2, 6, qc=chain[2].qc)
    bad_sig.round = 7
    bad_vote = messages.Vote(v.hash, 2, v.author, v.signature)
    outsider = messages.Vote(v.hash, 1, crypto.PublicKey(bytes(range(32))), v.signature)
    frames = [bc.propose(b) for b in chain + [blk_tc, bad_sig]] + [
        bc.vote(v), bc.vote(bad_vote), bc.vote(outsider), bc.timeout(fx.timeout(2, 9, chain[2].qc)), bc.timeout(fx.timeout(1, 4, messages.QC.genesis())),
        bc.tc_msg(fx.tc(7)), bc.tc_msg(fx.tc(8, hqs=((0, 3), (1, 5)))), bc.sync_request(fx.d(b"m"), fx.pks[1]), bc.vote(v)[:-9]]
    g = wire.ingest_frames(frames)
    groups = engine.verify_groups(g["preimages"], g["pre_off"], g["sig"], g["msg_idx"], g["group_idx"], len(frames), mode=g["mode"], pk=g["pk"])
    assert groups[0] and not groups[5] and not groups[7]        # the bad block and the bad vote reject: both outcomes are covered
    engine.committee_register(np.array([np.frombuffer(p.b, np.uint8) for p in fx.pks]))
    try:
        with engine.queue() as q:
            for j, fr in enumerate(frames):
                got = wire.submit_frame(q, fr)
                if g["info"][j]["kind"] in (wire.KIND_SYNC_REQUEST, wire.KIND_MALFORMED):
                    assert got is None
                    continue
                info, ticket = got
                assert info["kind"] == g["info"][j]["kind"]
                bits = q.wait(ticket)
                assert len(bits) == int((g["group_idx"] == j).sum()) and bits.all() == groups[j], j
    finally:
        _clear(engine)
