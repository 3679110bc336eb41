"""Ownership of the engine's CUDA resources.  In hs_engine.cu every buffer, stream, event and IPC mapping is held by one of the owner types
at the top of the host side, and only they create or release one (hs_host_alloc / hs_host_free hand pinned memory to the caller).  On the
GPU, one context walks every path that allocates, replaces or releases a resource, three times in one process, with the oracle's verdicts
after every step and every callback fired exactly once."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE = os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")
OWNERS_BEGIN, OWNERS_END = "// ---- resource owners", "// ---- end of resource owners"
RELEASE = re.compile(r"\b(cudaFree|cudaFreeHost|cudaStreamDestroy|cudaEventDestroy|cudaIpcCloseMemHandle|cudaHostGetDevicePointer)\b")
CREATE = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaHostAlloc|cudaStreamCreate\w*|cudaEventCreate\w*|cudaIpcOpenMemHandle)\b")


def _function_lines(lines, signature):
    """Line numbers of the function whose definition starts with `signature`, through its closing brace at column 0."""
    start = next(i for i, s in enumerate(lines) if s.startswith(signature))
    end = next(i for i in range(start, len(lines)) if lines[i].startswith("}"))
    return set(range(start, end + 1))


def test_resources_are_created_and_released_only_by_their_owners():
    with open(ENGINE) as f:
        lines = f.read().splitlines()
    marks = [i for i, s in enumerate(lines) if s.startswith((OWNERS_BEGIN, OWNERS_END))]
    assert len(marks) == 2, "the owner section is missing"
    caller_memory = _function_lines(lines, "void *hs_host_alloc(") | _function_lines(lines, "void hs_host_free(")
    outside = {}
    for i, s in enumerate(lines):
        if marks[0] < i < marks[1] or i in caller_memory:
            continue
        code = re.sub(r'"(\\.|[^"\\])*"', '""', s).split("//", 1)[0]  # calls, not error strings or comments
        for m in list(RELEASE.finditer(code)) + list(CREATE.finditer(code)):
            outside.setdefault(m.group(1), []).append(i + 1)
    assert not outside, "CUDA resources created or released outside the owner types (call: lines): %s" % outside


# ---- GPU: every configure and teardown path of one context, three times
COMMITTEE, FOREIGN = 48, 16  # committee keys, then keys that are never registered
SIG_ENTRIES = (1024, 4096, 0, 1024)  # on, resize, off, on
BATCH_SIZES = ((64, 64 << 10), (128, 128 << 10), (0, 0), (64, 64 << 10))  # on, resize, off, on
CERT_CACHE = 1 << 20


def _requests(oracle, keys, rng, foreign=False):
    """One request of each kind {name: (submit(q, callback) -> ticket, the oracle's verdicts)}; foreign: signed by unregistered keys."""
    from test_queue_msgs import make_req, want
    from test_queue_tickets import recs_of
    lo, hi = (COMMITTEE, COMMITTEE + FOREIGN) if foreign else (0, COMMITTEE)
    vote = make_req(oracle, keys, "vote", 5, rng, corrupt=0.3, key_lo=lo, key_hi=hi)
    block = make_req(oracle, keys, "block_tc", 30, rng, corrupt=0.1, key_lo=lo, key_hi=hi)
    tc = make_req(oracle, keys, "tc", 7, rng, corrupt=0.2, key_lo=lo, key_hi=hi)
    return {
        "submit": (lambda q, cb: q.submit(recs_of(vote), callback=cb), want(oracle, vote)),
        "group": (lambda q, cb: q.submit_group(recs_of(block), block["modes"], callback=cb), want(oracle, block)),
        "msgs": (lambda q, cb: q.submit_msgs(tc["pre"], tc["off"], tc["sig"], tc["pk"], tc["mi"], modes=tc["modes"], callback=cb), want(oracle, tc)),
    }


def _batch(oracle, keys, rng):
    from test_queue_batch import concat, expected
    from test_queue_msgs import make_req
    parts = [make_req(oracle, keys, "block_tc", 20, rng, corrupt=0.1, key_hi=COMMITTEE),
             make_req(oracle, keys, "vote", 3, rng, key_lo=COMMITTEE, key_hi=COMMITTEE + FOREIGN)]
    b = concat(parts)
    return (lambda q, cb: q.submit_batch(b["pre"], b["off"], b["sig"], b["pk"], b["mi"], b["gi"], b["n_groups"], modes=b["modes"], callback=cb),
            expected(oracle, parts))


def _check(q, reqs):
    """Submits every request and waits for it: the oracle's verdicts."""
    from test_queue_tickets import same
    tickets = {name: submit(q, None) for name, (submit, _) in reqs.items()}
    for name, t in tickets.items():
        assert t is not None and same(q.wait(t), reqs[name][1]), name


def _cached_qc(q, oracle, keys, rng):
    """Turns the certificate cache on and verifies a QC: an identical group later is answered from the cache.  Returns that request."""
    from test_queue_msgs import _sign, want
    from test_queue_tickets import recs_of
    q.cert_cache(CERT_CACHE)
    hot = _sign(oracle, keys, [rng.bytes(40)], np.zeros(12, np.uint32), np.ones(12, np.uint8), rng, key_hi=COMMITTEE)
    assert q.wait(q.submit_group(recs_of(hot), hot["modes"])).all()
    return (lambda q, cb: q.submit_group(recs_of(hot), hot["modes"], callback=cb)), want(oracle, hot)


def _in_flight(q, oracle, keys, rng, fired):
    """Requests of every kind with callbacks, not waited for: {ticket: verdicts}."""
    reqs = dict(_requests(oracle, keys, rng))
    reqs.update({"generic_" + k: v for k, v in _requests(oracle, keys, rng, foreign=True).items()})
    reqs["batch"] = _batch(oracle, keys, rng)
    reqs["cache_hit"] = _cached_qc(q, oracle, keys, rng)
    return {submit(q, fired): w for submit, w in reqs.values()}


def _fired_once(fired, tickets):
    from test_queue_tickets import same
    assert sorted(fired.calls) == sorted(tickets)
    for t, w in tickets.items():
        assert len(fired.calls[t]) == 1, t
        status, bits = fired.calls[t][0]
        assert status == 0 and same(bits, w), t


def _cycle(oracle, keys, rng):
    from hotstuff_b200 import Engine
    from test_queue_msgs import make_req, want
    from test_queue_tickets import Fired, recs_of
    _, pks = keys
    e = Engine(0, base_window=12, key_window=8)  # small comb tables: the footprint stays small on a shared device
    try:
        # a committee, then one of a different size
        assert e.committee_register(pks[:COMMITTEE]).all()
        assert e.committee_register(pks[:COMMITTEE - 8]).all()
        # without a committee, a pass's keys are learned: the key cache's buffers and tables
        e.committee_register(np.zeros((0, 32), np.uint8))
        r = make_req(oracle, keys, "tc", 96, rng, corrupt=0.1, key_hi=COMMITTEE)
        for _ in range(2):
            assert (e.verify_rec128(recs_of(r)) == want(oracle, r)).all()
        assert e.cached_keys > 0
        assert e.committee_register(pks[:COMMITTEE]).all()

        q, q2 = e.queue(), e.queue()
        _check(q, _requests(oracle, keys, rng))
        for entries in SIG_ENTRIES:
            q.sig_cache(entries)
            _check(q, _requests(oracle, keys, rng))
        for on in (True, False, True):
            q.generic(on)
            _check(q, _requests(oracle, keys, rng, foreign=True))
        for items, nbytes in BATCH_SIZES:
            q.batch(items, nbytes)
            if items:
                _check(q, {"batch": _batch(oracle, keys, rng)})
        hit, w = _cached_qc(q, oracle, keys, rng)
        _check(q, {"cache_hit": (hit, w)})

        buf = ctypes.create_string_buffer(64)
        for _ in range(2):  # the second call replaces the first call's buffer
            assert e.lib.hs_peer_setup(e.h, 0, 1, 64, buf) == 0, e.lib.hs_last_error(e.h)
            assert e.lib.hs_peer_bitmap(e.h) and e.lib.hs_peer_timed_out(e.h) == 0
        _check(q, _requests(oracle, keys, rng))

        # hs_queue_destroy with every kind in flight
        fired = Fired()
        tickets = _in_flight(q, oracle, keys, rng, fired)
        q.close()
        _fired_once(fired, tickets)

        # hs_ctx_destroy with the second queue still attached, configured like the first
        q2.sig_cache(SIG_ENTRIES[0])
        q2.generic(True)
        q2.batch(*BATCH_SIZES[0])
        fired = Fired()
        tickets = _in_flight(q2, oracle, keys, rng, fired)
        q2.h = None
        e._queues.remove(q2)
    finally:
        e.close()
    _fired_once(fired, tickets)


@pytest.mark.gpu
def test_every_configure_and_teardown_path_three_times(oracle):
    """Three cycles on fresh contexts of one process: committees of two sizes, key learning, the signature cache on / resized / off / on,
    the generic path on / off / on, the batch lane on / resized / off / on, the certificate cache, hs_peer_setup twice, then
    hs_queue_destroy and hs_ctx_destroy with requests of every kind in flight.  Free device memory is printed before and after each cycle
    (not asserted: the device is shared)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import build
    build.build_engine()
    rng = np.random.default_rng(5150)
    seeds = rng.integers(0, 256, size=(COMMITTEE + FOREIGN, 32), dtype=np.uint8)
    keys = (seeds, oracle.keygen_batch(seeds))
    free = [torch.cuda.mem_get_info(0)[0] >> 20]
    for _ in range(3):
        _cycle(oracle, keys, rng)
        free.append(torch.cuda.mem_get_info(0)[0] >> 20)
    print("free device memory (MiB) before the cycles, then after each: %s" % free)
