"""The verify queue's explain lane (hs_queue_explain, hs_queue_submit_explain, hs_queue_submit_explain_msgs) on the GPU.

Every mask the lane gives is checked byte for byte against hs_explain_rec128 on the same record (for the preimage form, the record built
with Digest = SHA-512(preimage)[..32]), on the sets of test_explain.py: the golden vectors with the 12 speccheck classes, every torsion
encoding as A and as R, S = l - 1, l and 2^256 - 1, and 3,000 single-bit mutations; plus preimages of several lengths.  Then the lane's
mechanics: request sizes up to its limit and across the arena's wrap, callback / poll / wait and the packed byte layout, coalescing of
concurrent requests, argument errors, lane off and resizing, isolation from the votes and their counters, the context's mutex and the
GPU share while a large request runs, an audit and a repair with the lane in flight, and destroy with requests in flight."""
import ctypes
import hashlib
import threading
import time

import numpy as np
import pytest

from oracle_api import make_adversarial, make_workload, to_rec128
from test_explain import Expect, _mismatches, golden_rec128, mutated_records, s_edge_records, torsion_records
from test_table_repair import POKE_FLAG, _engine, _keys, _poke, hooklib  # noqa: F401  (hooklib: the -DHS_TEST_HOOKS build, a fixture)

HS_ERR_ARG, HS_ERR_NOMEM = 2, 3
vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731


@pytest.fixture(scope="module")
def eng():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine, build
    build.build_engine()
    e = Engine(0, base_window=16)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sets(oracle, golden):
    """name -> records (n, 128)."""
    return {"golden": golden_rec128(golden), "torsion": torsion_records(oracle, golden), "s_edges": s_edge_records(oracle),
            "mutations": mutated_records(oracle, 3000), "adversarial": make_adversarial(oracle, 2000, seed=12)}


def _msgs_form(recs, preimages):
    """The preimage form of records whose Digests are SHA-512(preimages[i])[..32]: (pre, pre_off, sig, pk, msg_idx, records with Digests)."""
    pre = b"".join(preimages)
    off = np.zeros(len(preimages) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in preimages])
    dig = np.stack([np.frombuffer(hashlib.sha512(p).digest()[:32], np.uint8) for p in preimages])
    full = np.concatenate([recs[:, :96], dig], axis=1)
    return np.frombuffer(pre, np.uint8).copy(), off, recs[:, :64].copy(), recs[:, 64:96].copy(), np.arange(len(recs), dtype=np.uint32), full


def _explain_q(q, recs):
    return q.wait(q.submit_explain(recs))


@pytest.mark.gpu
def test_masks_equal_hs_explain_rec128_for_both_forms(eng, sets, golden, oracle):
    q = eng.queue()
    q.explain(8192, 4 << 20)
    expect = Expect(oracle)
    for name, recs in sets.items():
        want = eng.explain(recs)
        got = _explain_q(q, recs)
        assert got.dtype == np.uint8 and got.shape == want.shape
        assert not _mismatches(got, want), (name, _mismatches(got, want))
        assert (want == expect.recs(recs)).all(), name  # and both equal the oracle's masks
        for i in range(0, len(recs), max(1, len(recs) // 8)):  # one-record requests
            assert int(_explain_q(q, recs[i:i + 1])[0]) == int(want[i]), (name, i)
        # the preimage form: each record's 32-byte message becomes a preimage it signs the Digest of
        pre, off, sig, pk, mi, full = _msgs_form(recs, [r[96:].tobytes() for r in recs])
        got = q.wait(q.submit_explain_msgs(pre, off, sig, pk, mi))
        assert not _mismatches(got, eng.explain(full)), (name, "msgs")
    # every golden vector in the preimage form, speccheck classes included, over its own message (not only the 32-byte ones)
    vs = golden["vectors"]
    assert sum(v["group"] == "speccheck" for v in vs) == 12
    recs = np.stack([np.frombuffer(bytes.fromhex(v["sig"]) + bytes.fromhex(v["pk"]) + bytes(32), np.uint8) for v in vs])
    pre, off, sig, pk, mi, full = _msgs_form(recs, [bytes.fromhex(v["msg"]) for v in vs])
    assert (q.wait(q.submit_explain_msgs(pre, off, sig, pk, mi)) == eng.explain(full)).all()
    q.close()


@pytest.mark.gpu
def test_preimages_of_several_lengths_and_shared_preimages(eng, oracle):
    q = eng.queue()
    q.explain(4096, 4 << 20)
    rng = np.random.default_rng(71)
    lengths = [0, 1, 16, 40, 111, 112, 127, 128, 129, 239, 240, 256, 1000, 4096, 15000]
    preimages = [rng.bytes(n) for n in lengths]
    seeds = [rng.bytes(32) for _ in range(4)]
    rows, mi = [], []
    for k, p in enumerate(preimages):
        d = hashlib.sha512(p).digest()[:32]
        for j in range(3):  # three records per preimage: a valid signature, a flipped S bit, a signature over another Digest
            sd = seeds[(k + j) % 4]
            sig = bytearray(oracle.sign(sd, d if j != 2 else rng.bytes(32)))
            if j == 1:
                sig[40] ^= 2
            rows.append(np.frombuffer(bytes(sig) + oracle.keygen(sd) + d, np.uint8))
            mi.append(k)
    full = np.stack(rows)
    off = np.zeros(len(preimages) + 1, np.uint64)
    off[1:] = np.cumsum(lengths)
    pre = np.frombuffer(b"".join(preimages), np.uint8).copy()
    want = eng.explain(full)
    assert (want[0::3] == 0).all() and (want[2::3] != 0).all()
    got = q.wait(q.submit_explain_msgs(pre, off, full[:, :64], full[:, 64:96], np.array(mi, np.uint32)))
    assert not _mismatches(got, want), _mismatches(got, want)
    # records in another order than their preimages, and preimages no record names
    perm = rng.permutation(len(full))
    got = q.wait(q.submit_explain_msgs(pre, off, full[perm, :64], full[perm, 64:96], np.array(mi, np.uint32)[perm]))
    assert (got == want[perm]).all()
    q.close()


@pytest.mark.gpu
def test_request_sizes_up_to_the_limit_and_across_the_arena_wrap(eng, sets):
    recs = sets["mutations"]
    want = eng.explain(recs)
    q = eng.queue()
    limit = 1000
    q.explain(limit, limit * 128 + limit + 32)  # the largest Digest request fits exactly: arena 2^18 bytes, two such regions
    for n in (1, 2, 31, 500, limit):
        assert (_explain_q(q, recs[:n]) == want[:n]).all(), n
    from hotstuff_b200 import EngineError
    with pytest.raises(EngineError):  # one record over the limit: HS_ERR_ARG, not back-pressure
        q.submit_explain(recs[:limit + 1])
    q.close()


@pytest.mark.gpu
def test_requests_straddling_the_arena_wrap(eng, sets):
    recs = sets["mutations"]
    want = eng.explain(recs)
    q = eng.queue()
    q.explain(700, 700 * 128 + 700 + 32)  # arena 2^18 = 262,144 bytes
    rng = np.random.default_rng(73)
    pos = 0
    tickets = []
    for _ in range(40):  # regions of odd sizes walk the arena round several times; many wait together across its end
        n = int(rng.integers(1, 700))
        lo = int(rng.integers(0, len(recs) - n))
        t = q.submit_explain(recs[lo:lo + n])
        if t is None:  # the arena is full right now: back-pressure, then drain
            for tt, a, b in tickets:
                assert (q.wait(tt) == want[a:b]).all()
            tickets = []
            t = q.submit_explain(recs[lo:lo + n])
        tickets.append((t, lo, lo + n))
        pos += n * 128 + ((n + 15) & ~15) + 16
    for tt, a, b in tickets:
        assert (q.wait(tt) == want[a:b]).all()
    assert pos > 3 * (1 << 18)
    q.close()


@pytest.mark.gpu
def test_callback_poll_wait_and_the_packed_byte_layout(eng, sets):
    recs = sets["adversarial"]
    want = eng.explain(recs)
    q = eng.queue()
    q.explain(64, 64 * 128 + 64 + 32)
    lib = eng.lib
    for n in (1, 3, 4, 5):
        t = ctypes.c_size_t(0)
        assert lib.hs_queue_submit_explain(q.h, vp(recs[:n]), n, None, None, ctypes.byref(t)) == 0
        words = np.full((n + 3) // 4 + 2, 0xDEADBEEF, np.uint32)
        assert lib.hs_queue_wait(q.h, t.value, vp(words)) == 0
        w = (n + 3) // 4
        assert (words[w:] == 0xDEADBEEF).all(), n  # exactly (n + 3) / 4 words written
        packed = np.zeros(4 * w, np.uint8)
        packed[:n] = want[:n]
        assert (words[:w] == packed.view("<u4")).all(), n  # byte i little-endian = record i, unused bytes 0
    # poll until done
    t = q.submit_explain(recs[:50])
    got = None
    while got is None:
        got = q.poll(t)
    assert (got == want[:50]).all()
    # callback, on the queue's thread
    done = threading.Event()
    seen = []
    q.submit_explain(recs[10:60], callback=lambda ticket, status, why: (seen.append((status, why)), done.set()))
    assert done.wait(30)
    assert seen[0][0] == 0 and (seen[0][1] == want[10:60]).all()
    with pytest.raises(Exception):  # a ticket is read once
        q.wait(t)
    q.close()


@pytest.mark.gpu
def test_concurrent_requests_share_launches(eng, sets):
    recs = sets["mutations"]
    want = eng.explain(recs)
    q = eng.queue()
    q.explain(16, 1 << 16)  # an arena of 2^17 bytes: room for all 256 one-record regions at once
    errors = []

    def worker(k):
        try:
            mine = []
            for j in range(16):  # 16 threads x 16 one-record requests, submitted without waiting
                i = (k * 16 + j) * 7
                mine.append((q.submit_explain(recs[i:i + 1]), i))
            for t, i in mine:
                assert t is not None
                assert int(q.wait(t)[0]) == int(want[i])
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    th = [threading.Thread(target=worker, args=(k,)) for k in range(16)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    st = q.explain_stats()
    assert st["requests"] == 256 and st["records"] == 256, st
    assert 1 <= st["launches"] < 256, st
    q.close()


@pytest.mark.gpu
def test_argument_errors_write_nothing_lane_off_and_resizing_drains(eng, sets):
    recs = sets["adversarial"]
    lib = eng.lib
    q = eng.queue()
    t = ctypes.c_size_t(777)
    pre = np.zeros(64, np.uint8)
    off = np.array([0, 32, 64], np.uint64)
    sig, pk = recs[:4, :64].copy(), recs[:4, 64:96].copy()
    mi = np.zeros(4, np.uint32)
    # lane off (the default)
    assert lib.hs_queue_submit_explain(q.h, vp(recs), 4, None, None, ctypes.byref(t)) == HS_ERR_ARG and t.value == 777
    assert "explain lane is off" in eng.last_error
    assert lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(off), 2, vp(sig), vp(pk), vp(mi), 4, None, None, ctypes.byref(t)) == HS_ERR_ARG
    assert lib.hs_queue_explain(q.h, 16, 0) == HS_ERR_ARG and lib.hs_queue_explain(q.h, 0, 4096) == HS_ERR_ARG
    assert lib.hs_queue_explain(None, 16, 4096) == HS_ERR_ARG
    q.explain(16, 16 * 128 + 16 + 32)
    bad = [
        lambda: lib.hs_queue_submit_explain(q.h, vp(recs), 0, None, None, ctypes.byref(t)),         # n = 0
        lambda: lib.hs_queue_submit_explain(q.h, None, 4, None, None, ctypes.byref(t)),             # NULL recs
        lambda: lib.hs_queue_submit_explain(q.h, vp(recs), 17, None, None, ctypes.byref(t)),        # over max_records
        lambda: lib.hs_queue_submit_explain(None, vp(recs), 4, None, None, ctypes.byref(t)),
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(off), 0, vp(sig), vp(pk), vp(mi), 4, None, None, ctypes.byref(t)),
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(off), 2, vp(sig), vp(pk), vp(np.array([0, 2, 0, 0], np.uint32)), 4, None, None,
                                                 ctypes.byref(t)),                                  # msg_idx >= n_msgs
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(np.array([0, 40, 32], np.uint64)), 2, vp(sig), vp(pk), vp(mi), 4, None, None,
                                                 ctypes.byref(t)),                                  # decreasing offsets
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(np.array([8, 32, 64], np.uint64)), 2, vp(sig), vp(pk), vp(mi), 4, None, None,
                                                 ctypes.byref(t)),                                  # not starting at 0
        lambda: lib.hs_queue_submit_explain_msgs(q.h, None, vp(off), 2, vp(sig), vp(pk), vp(mi), 4, None, None, ctypes.byref(t)),
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(off), 2, None, vp(pk), vp(mi), 4, None, None, ctypes.byref(t)),
        lambda: lib.hs_queue_submit_explain_msgs(q.h, vp(pre), vp(off), 2, vp(sig), vp(pk), None, 4, None, None, ctypes.byref(t)),
    ]
    for k, call in enumerate(bad):
        assert call() == HS_ERR_ARG, k
        assert t.value == 777, k
    # a region over max_bytes: 16 records of preimage form with 2 KB of preimages
    big = np.zeros(2048, np.uint8)
    assert lib.hs_queue_submit_explain_msgs(q.h, vp(big), vp(np.array([0, 2048], np.uint64)), 1, vp(sig), vp(pk), vp(mi), 4, None, None,
                                            ctypes.byref(t)) == HS_ERR_ARG
    assert "limits" in eng.last_error and t.value == 777
    assert q.explain_stats() == {"launches": 0, "records": 0, "requests": 0}
    # resizing waits for the requests already submitted: their callbacks have fired when it returns
    fired = []
    q.explain(4096, 1 << 20)
    for k in range(8):
        q.submit_explain(recs[:512], callback=lambda ticket, status, why, k=k: fired.append((k, status)))
    q.explain(64, 64 * 128 + 64 + 32)
    assert sorted(fired) == [(k, 0) for k in range(8)]
    assert q.explain_stats()["requests"] == 8
    q.explain(0, 0)  # off again
    assert lib.hs_queue_submit_explain(q.h, vp(recs), 4, None, None, ctypes.byref(t)) == HS_ERR_ARG
    q.close()


def _burst(q, recs, explain_recs, explains_per_burst):
    """recs as one-record votes from 8 threads; meanwhile another thread submits explain_recs requests.  Returns the vote verdicts."""
    got = np.zeros(len(recs), bool)
    stop = threading.Event()
    xt = []

    def explainer():
        i = 0
        while not stop.is_set() and i < explains_per_burst:
            t = q.submit_explain(explain_recs[(i * 5) % len(explain_recs):][:5])
            if t is not None:
                xt.append(t)
            i += 1
            time.sleep(0.0005)

    def voter(k):
        ts = [(i, q.submit(recs[i:i + 1])) for i in range(k, len(recs), 8)]
        for i, t in ts:
            got[i] = q.wait(t)[0]
    th = [threading.Thread(target=voter, args=(k,)) for k in range(8)]
    ex = threading.Thread(target=explainer) if explains_per_burst else None
    if ex:
        ex.start()
    for x in th:
        x.start()
    for x in th:
        x.join()
    if ex:
        ex.join()
    for t in xt:
        q.wait(t)
    return got, len(xt)


@pytest.mark.gpu
def test_votes_with_explains_flowing_get_the_oracles_verdicts_and_the_same_counters(eng, oracle, sets):
    w = make_workload(oracle, 667, n_keys=128, seed=81, corrupt_frac=0.05)
    recs = to_rec128(w)
    want = oracle.verify_rec128(recs)
    eng.committee_register(w["pks"])
    junk = sets["adversarial"]
    counters = {}
    for explains in (0, 200):
        q = eng.queue()
        if explains:
            q.explain(64, 64 * 128 + 64 + 32)
        got, n_x = _burst(q, recs, junk, explains)
        assert (got == want).all(), np.nonzero(got != want)[0][:8]
        # one 667-record certificate: its launch count does not depend on how votes coalesce
        assert (np.asarray(q.wait(q.submit_group(recs))) == want).all()
        counters[explains] = (q.stats(), q.digest_stats(), q.generic_stats(), q.batch_stats(), q.cert_stats(), q.sig_stats())
        if explains:
            assert n_x > 0 and q.explain_stats()["requests"] == n_x
        q.close()
    (s0, *rest0), (s1, *rest1) = counters[0], counters[200]
    assert rest0 == rest1
    # bulk and slow-path counts are the burst's (a record with a corrupted key takes the slow path); how many small launches the votes
    # shared, and so how many slow-path records rode in them, depends on how they coalesced, with or without explains
    for k in ("bulk_launches", "bulk_records", "slow_requests", "slow_records"):
        assert s0[k] == s1[k], (k, s0, s1)
    for s in (s0, s1):
        assert 1 <= s["small_launches"] <= 668 and s["small_records"] <= 2 * 667, s


@pytest.mark.gpu
def test_a_large_explain_request_holds_neither_the_mutex_nor_the_gpu(eng, oracle, sets):
    w = make_workload(oracle, 64, n_keys=16, seed=91)
    small = to_rec128(w)
    eng.committee_register(w["pks"])
    q = eng.queue()
    q.explain(65536, 65536 * 128 + 65536 + 32)
    big = np.tile(sets["mutations"], (22, 1))[:65536]
    want_big = np.tile(eng.explain(sets["mutations"]), 22)[:65536]
    stamps = {}
    done = threading.Event()

    def on_explain(ticket, status, why):
        stamps["explain"] = time.perf_counter()
        stamps["why"] = (status, why)
        done.set()
    q.submit_explain(big, callback=on_explain)
    time.sleep(0.002)  # the launch is enqueued and running

    def sync_verify():
        ok = eng.verify_rec128(small[:1])
        stamps["sync"] = time.perf_counter()
        stamps["sync_ok"] = bool(ok[0])
    th = threading.Thread(target=sync_verify)
    th.start()
    t = q.submit(small[1:2])
    ok = q.wait(t)
    stamps["queue"] = time.perf_counter()
    th.join()
    assert done.wait(120)
    assert stamps["sync_ok"] and bool(ok[0])
    assert stamps["sync"] < stamps["explain"] and stamps["queue"] < stamps["explain"], stamps
    assert q.stats()["small_launches"] >= 1  # the queue request ran k_verify_small
    status, why = stamps["why"]
    assert status == 0 and not _mismatches(why, want_big)
    assert q.explain_stats() == {"launches": 1, "records": 65536, "requests": 1}
    q.close()


@pytest.mark.gpu
def test_an_audit_and_a_repair_with_the_lane_in_flight_leave_the_masks_unchanged(hooklib, oracle, sets):
    e = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _keys(e, 32, seed=95)
        assert e.committee_register(pks).all()
        recs = np.tile(np.concatenate([sets["mutations"], sets["torsion"], sets["s_edges"]]), (6, 1))
        want = e.explain(recs)
        _poke(e, POKE_FLAG, 7, 0, 0x01)  # a finding for the repair to fix
        q = e.queue()
        q.explain(len(recs), len(recs) * 129 + 64)
        t = q.submit_explain(recs)
        failed, slot_bits = e.table_audit(expect=pks)
        assert failed and slot_bits[7]
        t2 = q.submit_explain(recs[: len(recs) // 2])
        found, failed, slot_bits = e.table_repair(expect=pks)
        assert found and failed == 0 and slot_bits[7]
        assert (q.wait(t) == want).all() and (q.wait(t2) == want[: len(recs) // 2]).all()
        assert (q.wait(q.submit_explain(recs[:100])) == want[:100]).all()
        q.close()
    finally:
        e.close()


@pytest.mark.gpu
def test_destroy_with_requests_in_flight_fires_every_callback(eng, sets):
    recs = sets["mutations"]
    want = eng.explain(recs)
    q = eng.queue()
    q.explain(3000, 3000 * 129 + 64)
    fired = []
    lock = threading.Lock()

    def cb(ticket, status, why, k=None):
        with lock:
            fired.append((status, why.copy()))
    submitted = [k for k in range(12) if q.submit_explain(recs[k * 200:k * 200 + 1000], callback=cb) is not None]
    assert len(submitted) >= 2
    q.close()  # completes every request in flight
    assert len(fired) == len(submitted)
    assert all(s == 0 for s, _ in fired)
    assert sorted(tuple(w) for _, w in fired) == sorted(tuple(want[k * 200:k * 200 + 1000]) for k in submitted)
