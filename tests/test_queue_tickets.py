"""The ticket contract of the verify queue across request kinds, on one queue with the certificate cache and the batch lane on and a
committee registered: hs_queue_submit, hs_queue_submit_group through the certificate cache, an identical group answered entirely from
the cache, hs_queue_submit_msgs and hs_queue_submit_batch share one ticket sequence, and each of their tickets is read exactly once,
by poll / wait or by its callback, as the header promises for every kind."""
import hashlib
import threading

import numpy as np
import pytest

from test_queue import _threads
from test_queue_batch import concat, expected
from test_queue_msgs import K, _clear, _register, _sign, make_req, want

pytestmark = pytest.mark.gpu
CACHE = 16 << 20
BATCH_ITEMS, BATCH_BYTES = 64, 64 << 10


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(9300)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture()
def committee(engine, keys):
    _register(engine, keys[1])
    yield
    _clear(engine)


def recs_of(r):
    """A preimage request as rec128 records over SHA-512(preimage)[..32]."""
    pre, off = r["pre"].tobytes(), r["off"]
    dig = np.array([np.frombuffer(hashlib.sha512(pre[int(off[j]):int(off[j + 1])]).digest()[:32], np.uint8) for j in range(len(off) - 1)])
    recs = np.zeros((len(r["mi"]), 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = r["sig"], r["pk"], dig[r["mi"]]
    return recs


def configure(q, oracle, keys, rng):
    """Turns the certificate cache and the batch lane on and puts a verified QC in the cache (one ticket).  Returns that QC as a
    request: all its records are one batch-eq span, so an identical group is answered entirely from the cache."""
    q.cert_cache(CACHE)
    q.batch(BATCH_ITEMS, BATCH_BYTES)
    hot = _sign(oracle, keys, [rng.bytes(40)], np.zeros(12, np.uint32), np.ones(12, np.uint8), rng)
    assert q.wait(q.submit_group(recs_of(hot), hot["modes"])).all()
    return hot


def kinds(q, oracle, keys, rng, hot):
    """One request of each kind: {name: (submit(callback) -> ticket, a submit of the same kind refused with HS_ERR_ARG, the
    oracle's verdicts)}, in submission order."""
    vote = make_req(oracle, keys, "vote", 5, rng, corrupt=0.3)
    block = make_req(oracle, keys, "block_tc", 30, rng, corrupt=0.1)
    tc = make_req(oracle, keys, "tc", 7, rng, corrupt=0.2)
    parts = [make_req(oracle, keys, "block_tc", 20, rng, corrupt=0.1), make_req(oracle, keys, "vote", 3, rng)]
    b, over = concat(parts), concat([make_req(oracle, keys, "tc", BATCH_ITEMS + 1, rng)])
    bad_modes = block["modes"].copy()
    bad_modes[3] = 2
    no_recs = dict(tc, **{k: tc[k][:0] for k in ("sig", "pk", "mi", "modes")})

    def msgs(r, cb=None):
        return q.submit_msgs(r["pre"], r["off"], r["sig"], r["pk"], r["mi"], modes=r["modes"], callback=cb)

    def batch(x, cb=None):
        return q.submit_batch(x["pre"], x["off"], x["sig"], x["pk"], x["mi"], x["gi"], x["n_groups"], modes=x["modes"], callback=cb)

    return {
        "submit": (lambda cb: q.submit(recs_of(vote), callback=cb), lambda: q.submit(recs_of(vote), mode=2), want(oracle, vote)),
        "group": (lambda cb: q.submit_group(recs_of(block), block["modes"], callback=cb),
                  lambda: q.submit_group(recs_of(block), bad_modes), want(oracle, block)),
        "cache_hit": (lambda cb: q.submit_group(recs_of(hot), hot["modes"], callback=cb),
                      lambda: q.submit_group(recs_of(hot)[:0]), want(oracle, hot)),
        "msgs": (lambda cb: msgs(tc, cb), lambda: msgs(no_recs), want(oracle, tc)),
        "batch": (lambda cb: batch(b, cb), lambda: batch(over), expected(oracle, parts)),
    }


def same(got, w):
    if isinstance(w, tuple):  # a batch ticket: (group bools, item bools)
        return len(got) == 2 and all(len(g) == len(x) and (g == x).all() for g, x in zip(got, w))
    return len(got) == len(w) and (got == w).all()


class Fired:
    """Callbacks by ticket: every call is kept, so a second call is seen."""

    def __init__(self):
        self.calls, self.cv = {}, threading.Condition()

    def __call__(self, ticket, status, bits):
        with self.cv:
            self.calls.setdefault(ticket, []).append((status, bits))
            self.cv.notify_all()

    def wait_for(self, tickets):
        with self.cv:
            assert self.cv.wait_for(lambda: all(t in self.calls for t in tickets), timeout=60)


@pytest.mark.parametrize("read", ["wait", "poll", "callback"])
def test_one_ticket_sequence_and_one_read_per_ticket(engine, oracle, keys, committee, read):
    """Tickets of all kinds go up by exactly one in submission order, from 1; a refused submit of each kind between them takes no
    number.  Every ticket is read once: by wait (a second wait or a poll is HS_ERR_ARG), by poll until done (a wait afterwards is
    HS_ERR_ARG), or by its callback (the ticket is not readable and the callback fires once), with the oracle's verdicts."""
    from hotstuff_b200 import EngineError
    rng = np.random.default_rng({"wait": 1, "poll": 2, "callback": 3}[read])
    with engine.queue() as q:
        hot = configure(q, oracle, keys, rng)
        ks = kinds(q, oracle, keys, rng, hot)
        fired = Fired()
        tickets = {}
        for name, (submit, refused, _) in ks.items():
            with pytest.raises(EngineError, match="status 2"):
                refused()
            hits = q.cert_stats()["hits"]
            tickets[name] = submit(fired if read == "callback" else None)
            if name == "cache_hit":  # answered entirely from the cache
                assert q.cert_stats()["hits"] == hits + 1
        assert list(tickets.values()) == [2, 3, 4, 5, 6]  # ticket 1 is configure's QC
        for name, t in tickets.items():
            w = ks[name][2]
            if read == "wait":
                assert same(q.wait(t), w), name
                for again in (q.wait, q.poll):
                    with pytest.raises(EngineError, match="status 2"):
                        again(t)
            elif read == "poll":
                while (got := q.poll(t)) is None:
                    threading.Event().wait(0.0002)
                assert same(got, w), name
                with pytest.raises(EngineError, match="status 2"):
                    q.wait(t)
            else:
                for read_it in (q.wait, q.poll):
                    with pytest.raises(EngineError, match="status 2"):
                        read_it(t)
        if read == "callback":
            fired.wait_for(tickets.values())
    if read == "callback":  # the queue is closed: nothing fires late
        assert sorted(fired.calls) == sorted(tickets.values())
        for name, t in tickets.items():
            assert len(fired.calls[t]) == 1, name
            status, bits = fired.calls[t][0]
            assert status == 0 and same(bits, ks[name][2]), name


def test_close_fires_every_kind_once(engine, oracle, keys, committee):
    """Requests of all five kinds in flight with callbacks when the queue is closed: every callback fires exactly once with the
    oracle's verdicts, and no thread is left."""
    rng = np.random.default_rng(4)
    with engine.queue() as q:  # the lane's first streams and the first queue: lets the CUDA runtime settle its own threads
        hot = configure(q, oracle, keys, rng)
        for submit, _, _ in kinds(q, oracle, keys, rng, hot).values():
            submit(None)
    before = _threads()
    q = engine.queue()
    hot = configure(q, oracle, keys, rng)
    ks = kinds(q, oracle, keys, rng, hot)
    fired = Fired()
    tickets = {name: submit(fired) for name, (submit, _, _) in ks.items()}
    q.close()
    assert sorted(fired.calls) == sorted(tickets.values())
    for name, t in tickets.items():
        assert len(fired.calls[t]) == 1, name
        status, bits = fired.calls[t][0]
        assert status == 0 and same(bits, ks[name][2]), name
    assert _threads() == before
