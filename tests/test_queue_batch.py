"""The verify queue's batch lane (hs_queue_batch / hs_queue_submit_batch, VerifyQueue.batch / submit_batch): a whole hs_verify_groups
pass as one non-blocking request on the lane's own stream and scratch.  Group and item bits must equal hs_verify_groups on the same
arrays and the oracle's per-item verdicts, with or without a registered committee and with keys outside it, while the ring's
requests and the synchronous entry points run on the same context."""
import hashlib
import struct
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial
from test_queue_msgs import K, _clear, _register, _sign, make_req, want

pytestmark = pytest.mark.gpu
MAX_ITEMS, MAX_BYTES = 8192, 4 << 20


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(9100)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture(scope="module")
def foreign(oracle):
    """64 keys that are never registered."""
    rng = np.random.default_rng(9101)
    seeds = rng.integers(0, 256, size=(64, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture()
def committee(engine, keys):
    _register(engine, keys[1])
    yield
    _clear(engine)


@pytest.fixture()
def no_committee(engine):
    _clear(engine)
    yield
    _clear(engine)


def adversarial_req(oracle, rng, n):
    """make_adversarial's (sig, pk) pairs, each over its own random preimage, in random modes."""
    adv = make_adversarial(oracle, n, seed=int(rng.integers(1 << 30)))
    pres = [rng.bytes(int(rng.integers(0, 200))) for _ in range(n)]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in pres])
    return dict(pre=np.frombuffer(b"".join(pres), np.uint8).copy(), off=off, sig=adv[:, :64].copy(), pk=adv[:, 64:96].copy(),
                mi=np.arange(n, dtype=np.uint32), modes=rng.integers(0, 2, n).astype(np.uint8))


def concat(reqs, extra_groups=0):
    """One batch: request g is group g (extra_groups empty groups after them)."""
    pre, offs, mi, gi = [], [np.zeros(1, np.uint64)], [], []
    nb = nm = 0
    for g, r in enumerate(reqs):
        pre.append(r["pre"])
        offs.append(r["off"][1:] + nb)
        mi.append(r["mi"] + nm)
        gi.append(np.full(len(r["mi"]), g, np.uint32))
        nb += int(r["off"][-1])
        nm += len(r["off"]) - 1
    cat = lambda k: np.concatenate([r[k] for r in reqs])
    return dict(pre=np.concatenate(pre).astype(np.uint8), off=np.concatenate(offs).astype(np.uint64), sig=cat("sig"), pk=cat("pk"),
                mi=np.concatenate(mi).astype(np.uint32), gi=np.concatenate(gi), modes=cat("modes"), n_groups=len(reqs) + extra_groups)


def expected(oracle, reqs, extra_groups=0):
    items = [want(oracle, r) for r in reqs]
    return np.array([x.all() for x in items] + [True] * extra_groups), np.concatenate(items)


def submit(q, b, callback=None, modes=True):
    while (t := q.submit_batch(b["pre"], b["off"], b["sig"], b["pk"], b["mi"], b["gi"], b["n_groups"], modes=b["modes"] if modes else None,
                               callback=callback)) is None:
        threading.Event().wait(0.0005)  # no room now: back-pressure
    return t


def sync(engine, b):
    return engine.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"], pk=b["pk"], want_items=True)


def mixed(oracle, keys, rng, n_certs, vote_n, foreign=None, foreign_frac=0.0):
    """Blocks (author + QC + TC), Timeouts, TCs and votes of about vote_n signatures each, 1.5 % corrupted; `foreign_frac` of them
    signed by foreign keys; and one request of adversarial records."""
    reqs = []
    for k in range(n_certs):
        shape = ("block_tc", "timeout", "tc", "vote")[k % 4]
        n = 1 if shape == "vote" and k % 8 == 3 else max(2, int(rng.integers(vote_n // 2, vote_n + 1)))
        ks = foreign if foreign is not None and rng.random() < foreign_frac else keys
        reqs.append(make_req(oracle, ks, shape, n, rng, corrupt=0.015, key_hi=len(ks[1])))
    reqs.append(adversarial_req(oracle, rng, 96))
    return reqs


def outside(b, members):
    """Items whose key is not one of `members`."""
    return int(np.isin(b["pk"].view("V32").ravel(), np.ascontiguousarray(members).view("V32").ravel(), invert=True).sum())


def check(engine, oracle, q, reqs, extra_groups=0):
    b = concat(reqs, extra_groups)
    g_want, i_want = expected(oracle, reqs, extra_groups)
    g, items = q.wait(submit(q, b))
    sg, si = sync(engine, b)
    assert (items == si).all() and (g == sg).all()
    assert (items == i_want).all() and (g == g_want).all()
    return b


@pytest.mark.parametrize("setup", ["committee", "outside", "none"])
def test_parity_with_verify_groups_and_the_oracle(engine, oracle, keys, foreign, setup):
    """Batches from 1 to about 7,000 items: every group and item bit equals hs_verify_groups and the oracle, with a registered
    committee, with some certificates signed by keys outside it, and with no committee at all (smaller batches)."""
    rng = np.random.default_rng({"committee": 1, "outside": 2, "none": 3}[setup])
    if setup == "none":
        _clear(engine)
        plan = [(1, 1), (3, 20), (12, 60), (24, 80)]
    else:
        _register(engine, keys[1])
        plan = [(1, 1), (4, 30), (16, 100), (40, 150), (14, 670)]
    try:
        with engine.queue() as q:
            q.batch(MAX_ITEMS, MAX_BYTES)
            for n_certs, vote_n in plan:
                if n_certs == 1:  # a single item
                    reqs = [make_req(oracle, keys, "vote", 1, rng)]
                else:
                    reqs = mixed(oracle, keys, rng, n_certs, vote_n, foreign, 0.3 if setup == "outside" else 0.0)
                b = check(engine, oracle, q, reqs)
            assert len(b["sig"]) > (4000 if setup != "none" else 800)
    finally:
        _clear(engine)


def test_edge_shapes(engine, oracle, keys, committee):
    """Empty groups, preimages no item names, zero-length and 15 KB preimages, the same record under both modes, no modes array."""
    rng = np.random.default_rng(5)
    with engine.queue() as q:
        q.batch(MAX_ITEMS, MAX_BYTES)
        seeds, pks = keys
        zero = _sign(oracle, keys, [b"", rng.bytes(15 * 1024), b"", rng.bytes(7)], np.array([0, 1, 1, 2], np.uint32), np.array([0, 1, 0, 0], np.uint8), rng)
        both = _sign(oracle, keys, [rng.bytes(40)], np.zeros(2, np.uint32), np.array([0, 1], np.uint8), rng)
        both["sig"][1], both["pk"][1] = both["sig"][0], both["pk"][0]
        small = make_req(oracle, keys, "timeout", 5, rng)   # carries a preimage no record names
        reqs = [zero, both, small, make_req(oracle, keys, "block_tc", 30, rng)]
        check(engine, oracle, q, reqs, extra_groups=37)
        # empty groups between the filled ones: group 2k + 1 has no items and reads 1
        b = concat(reqs)
        b["gi"] = b["gi"] * 2
        b["n_groups"] = 2 * len(reqs) + 1
        g, items = q.wait(submit(q, b))
        sg, si = engine.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"], pk=b["pk"], want_items=True)
        assert (g == sg).all() and (items == si).all() and g[1::2].all()
        # modes omitted: every item strict
        b = concat([make_req(oracle, keys, "tc", 40, rng), both])
        g, items = q.wait(submit(q, b, modes=False))
        sg, si = engine.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], pk=b["pk"], want_items=True)
        assert (g == sg).all() and (items == si).all() and items[-1] == items[-2]


def test_argument_errors_and_back_pressure(engine, oracle, keys, committee):
    """Every HS_ERR_ARG case of hs_queue_submit_batch, and HS_ERR_NOMEM reached deterministically: while the dispatcher thread is held
    in a callback, submitted requests keep their arena regions, so the arena fills; after the callback returns they complete and a
    resubmit is accepted."""
    from hotstuff_b200 import EngineError
    rng = np.random.default_rng(6)
    b = concat([make_req(oracle, keys, "block_tc", 20, rng), make_req(oracle, keys, "vote", 3, rng)])
    with engine.queue() as q:
        with pytest.raises(EngineError, match="status 2"):
            submit(q, b)                                   # the lane is off
        q.batch(64, 64 << 10)

        def bad(**kw):
            x = dict(b, **kw)
            with pytest.raises(EngineError, match="status 2"):
                q.submit_batch(x["pre"], x["off"], x["sig"], x["pk"], x["mi"], x["gi"], x["n_groups"], modes=x["modes"])

        bad(sig=b["sig"][:0], pk=b["pk"][:0], mi=b["mi"][:0], gi=b["gi"][:0], modes=b["modes"][:0])   # no items
        bad(n_groups=0)
        off = b["off"].copy()
        off[1], off[2] = off[2], off[1]
        bad(off=off)                                                                                  # decreasing offsets
        bad(off=b["off"] + 1)                                                                         # off[0] != 0
        bad(mi=np.where(np.arange(len(b["mi"])) == 3, len(b["off"]) - 1, b["mi"]).astype(np.uint32))   # msg_idx >= n_msgs
        bad(gi=np.where(np.arange(len(b["gi"])) == 5, 2, b["gi"]).astype(np.uint32))                 # group_idx >= n_groups
        bad(modes=np.where(np.arange(len(b["modes"])) == 0, 2, b["modes"]).astype(np.uint8))          # a mode byte > 1
        big = concat([make_req(oracle, keys, "tc", 65, rng)])
        bad(**big)                                                                                    # more items than the lane takes
        huge = concat([_sign(oracle, keys, [rng.bytes(70000)], np.zeros(1, np.uint32), np.zeros(1, np.uint8), rng)])
        bad(**huge)                                                                                   # more bytes than the lane takes
        with pytest.raises(EngineError, match="status 2"):
            q.batch(64, 0)
        # back-pressure: hold the dispatcher in the first request's callback
        first_req = make_req(oracle, keys, "vote", 1, rng)
        g_want, i_want = expected(oracle, [first_req])
        first = concat([first_req])
        entered, release, got = threading.Event(), threading.Event(), []

        def hold(ticket, status, bits):
            got.append((status, bits))
            entered.set()
            release.wait(60)

        submit(q, first, callback=hold)
        assert entered.wait(60)
        fill_req = _sign(oracle, keys, [rng.bytes(20000)], np.zeros(1, np.uint32), np.zeros(1, np.uint8), rng)
        fill_want = want(oracle, fill_req)
        fill = concat([fill_req])
        tickets = []
        for _ in range(16):
            t = q.submit_batch(fill["pre"], fill["off"], fill["sig"], fill["pk"], fill["mi"], fill["gi"], 1, modes=fill["modes"])
            if t is None:
                break
            tickets.append(t)
        assert t is None and 1 <= len(tickets) < 16
        release.set()
        assert got[0][0] == 0 and (got[0][1][0] == g_want).all() and (got[0][1][1] == i_want).all()
        for t in tickets:
            g, items = q.wait(t)
            assert (items == fill_want).all() and g[0] == fill_want[0]
        t = q.submit_batch(fill["pre"], fill["off"], fill["sig"], fill["pk"], fill["mi"], fill["gi"], 1, modes=fill["modes"])
        assert t is not None and (q.wait(t)[1] == fill_want).all()


def test_concurrency_with_votes_and_synchronous_calls(engine, oracle, keys, foreign, committee):
    """16 threads submit votes through the ring, one thread submits batches and one calls hs_verify_groups / hs_verify_tcs on the same
    context: every verdict is the oracle's, so the lane's scratch is its own."""
    rng = np.random.default_rng(8)
    seeds, pks = keys
    votes = []
    for t in range(16):
        votes.append([make_req(oracle, keys, "vote", 1, np.random.default_rng(100 * t + k), corrupt=0.1) for k in range(25)])
    batches = [mixed(oracle, keys, rng, 12, 120, foreign, 0.2) for _ in range(6)]
    sync_reqs = [mixed(oracle, keys, rng, 8, 200, foreign, 0.2) for _ in range(6)]
    tr = rng.integers(1, 1 << 40, 300).astype(np.uint64)
    hq = rng.integers(1, 1 << 40, 300).astype(np.uint64)
    tcs = _sign(oracle, keys, [struct.pack("<QQ", int(a), int(b_)) for a, b_ in zip(tr, hq)], np.arange(300, dtype=np.uint32), np.zeros(300, np.uint8), rng,
                corrupt=0.05)
    tc_want = want(oracle, tcs)
    errors = []

    def guard(fn):
        def run():
            try:
                fn()
            except BaseException as e:  # reported below
                errors.append(e)
        return run

    with engine.queue() as q:
        q.batch(MAX_ITEMS, MAX_BYTES)

        def voter(t):
            for r in votes[t]:
                w = want(oracle, r)
                recs = np.zeros((1, 128), np.uint8)
                recs[:, :64], recs[:, 64:96] = r["sig"], r["pk"]
                recs[:, 96:] = np.frombuffer(hashlib.sha512(r["pre"].tobytes()[int(r["off"][0]):int(r["off"][1])]).digest()[:32], np.uint8)
                while (tk := q.submit(recs)) is None:
                    threading.Event().wait(0.0005)
                assert (q.wait(tk) == w).all()

        def batcher():
            for reqs in batches:
                g_want, i_want = expected(oracle, reqs)
                g, items = q.wait(submit(q, concat(reqs)))
                assert (g == g_want).all() and (items == i_want).all()

        def syncer():
            for reqs in sync_reqs:
                g_want, i_want = expected(oracle, reqs)
                g, items = sync(engine, concat(reqs))
                assert (g == g_want).all() and (items == i_want).all()
                assert (engine.verify_tcs(tr, tcs["sig"], hq, pk=tcs["pk"]) == tc_want).all()

        ths = [threading.Thread(target=guard(lambda t=t: voter(t))) for t in range(16)] + [threading.Thread(target=guard(batcher)),
                                                                                           threading.Thread(target=guard(syncer))]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
    assert not errors, errors[:3]


def test_committee_changes_between_batches(engine, oracle, keys, foreign):
    """hs_committee_register and hs_committee_update between batches: verdicts stay the oracle's, and the outside-committee count
    follows the committee."""
    rng = np.random.default_rng(9)
    try:
        with engine.queue() as q:
            q.batch(MAX_ITEMS, MAX_BYTES)
            reqs = mixed(oracle, keys, rng, 10, 100, foreign, 0.3)
            b = concat(reqs)
            for step in range(4):
                if step == 0:
                    _register(engine, keys[1])
                    members = np.unique(keys[1], axis=0)
                elif step == 1:
                    removed = members[:64]
                    engine.committee_update(add=foreign[1][:32], remove=np.arange(0, 64, dtype=np.uint32))
                    members = np.concatenate([members[64:], foreign[1][:32]])
                    assert not np.isin(removed.view("V32").ravel(), members.view("V32").ravel()).any()
                elif step == 2:
                    _register(engine, np.concatenate([keys[1], foreign[1]]))
                    members = np.concatenate([keys[1], foreign[1]])
                else:
                    _clear(engine)
                    members = np.zeros((0, 32), np.uint8)
                before = q.batch_stats()["outside_committee"]
                check(engine, oracle, q, reqs)
                assert q.batch_stats()["outside_committee"] - before == (outside(b, members) if len(members) else len(b["sig"]))
    finally:
        _clear(engine)


def test_destroy_with_batches_pending_fires_every_callback(engine, oracle, keys, committee):
    rng = np.random.default_rng(10)
    batches = [concat(mixed(oracle, keys, rng, 6, 200)) for _ in range(6)]
    expect = {k: sync(engine, b) for k, b in enumerate(batches)}
    fired = {}
    lock = threading.Lock()
    q = engine.queue()
    q.batch(MAX_ITEMS, MAX_BYTES)
    for k, b in enumerate(batches):
        def cb(ticket, status, bits, k=k):
            with lock:
                fired.setdefault(k, []).append((status, bits))
        submit(q, b, callback=cb)
    q.close()
    assert sorted(fired) == list(range(len(batches))) and all(len(v) == 1 for v in fired.values())
    for k, v in fired.items():
        status, (g, items) = v[0]
        assert status == 0 and (g == expect[k][0]).all() and (items == expect[k][1]).all()


def test_counters(engine, oracle, keys, foreign, committee):
    """hs_queue_batch_stats counts exactly; the ring's counters do not move; each pass is six launches with the committee's table path
    (digest, lookup, miss pass, main, finish, k_batch_done) and four without a committee."""
    rng = np.random.default_rng(11)
    with engine.queue() as q:
        q.batch(MAX_ITEMS, MAX_BYTES)
        q.cert_cache(1 << 20)
        q.sig_cache(4096)
        q.generic(True)
        others = (q.stats(), q.digest_stats(), q.cert_stats(), q.sig_stats(), q.generic_stats())
        total = dict(passes=0, items=0, groups=0, preimage_bytes=0, outside_committee=0)
        for k in range(3):
            reqs = mixed(oracle, keys, rng, 8, 50, foreign, 0.4)
            b = concat(reqs, extra_groups=k)
            launches = engine.kernel_launches
            q.wait(submit(q, b))
            assert engine.kernel_launches - launches == 6
            total["passes"] += 1
            total["items"] += len(b["sig"])
            total["groups"] += b["n_groups"]
            total["preimage_bytes"] += int(b["off"][-1])
            total["outside_committee"] += outside(b, keys[1])
            assert q.batch_stats() == total
        assert (q.stats(), q.digest_stats(), q.cert_stats(), q.sig_stats(), q.generic_stats()) == others
        _clear(engine)
        b = concat([make_req(oracle, keys, "timeout", 20, rng)])
        launches = engine.kernel_launches
        q.wait(submit(q, b))
        assert engine.kernel_launches - launches == 4
        assert q.batch_stats()["outside_committee"] == total["outside_committee"] + 20


def test_frames_through_the_lane_equal_verify_frames(engine, oracle, golden):
    """wire.verify_frames_queued equals wire.verify_frames on the scenario frames, malformed frames included, and wire.submit_frames
    gives one group per frame."""
    import bincode_ref as bc
    import messages_scenarios as sc
    from hotstuff_b200 import crypto, messages, wire
    from test_wire_ingest import _messages
    fx = sc.Fixtures(oracle, golden, engine)
    chain, blk_tc, v, to, to_gen = _messages(fx)
    bad_sig = fx.block(2, 6, qc=chain[2].qc)
    bad_sig.round = 7
    reuse = fx.block(0, 6, qc=fx.qc_for(fx.d(b"y"), 5))
    reuse.qc.votes[1] = reuse.qc.votes[0]
    bad_vote = messages.Vote(v.hash, 2, v.author, v.signature)
    short_tc = fx.tc(8, hqs=((0, 3), (1, 5)))
    outsider = messages.Vote(v.hash, 1, crypto.PublicKey(bytes(range(32))), v.signature)
    good = bc.propose(blk_tc)
    frames = [bc.propose(b) for b in chain + [blk_tc, bad_sig, reuse]] + [
        bc.vote(v), bc.vote(bad_vote), bc.vote(outsider), bc.timeout(to), bc.timeout(to_gen), bc.tc_msg(fx.tc(7)), bc.tc_msg(short_tc),
        bc.sync_request(fx.d(b"m"), fx.pks[1]), good[:40], b"\x05\x00\x00\x00" + good[4:], b"", good + b"trailing"]
    want_ = wire.verify_frames(frames, fx.committee, engine)
    assert "Malformed" in want_ and "InvalidSignature" in want_ and None in want_
    with engine.queue() as q:
        q.batch(MAX_ITEMS, MAX_BYTES)
        assert wire.verify_frames_queued(frames, fx.committee, q) == want_
        for with_committee in (False, True):
            if with_committee:
                engine.committee_register(np.array([np.frombuffer(p.b, np.uint8) for p in fx.pks]))
            try:
                g, t = wire.submit_frames(q, frames)
                groups, items = q.wait(t)
                sg, si = engine.verify_groups(g["preimages"], g["pre_off"], g["sig"], g["msg_idx"], g["group_idx"], len(frames), mode=g["mode"], pk=g["pk"],
                                              want_items=True)
                assert (groups == sg).all() and (items == si).all() and len(groups) == len(frames)
            finally:
                _clear(engine)
        assert wire.submit_frames(q, [bc.sync_request(fx.d(b"m"), fx.pks[1]), b""])[1] is None
