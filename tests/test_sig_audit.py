"""The audit of the verify queue's signature cache (hs_queue_sig_audit, VerifyQueue.sig_audit) and its scrub slice (hs_scrub_sig_cache),
on the engine built with the corruption hooks (hs_test_poke_sig, -DHS_TEST_HOOKS): a stored flag byte or record word is changed in HBM,
the poke is shown to change verdicts, and one audit puts back exactly the byte a verify writes for the stored bytes.  Every verdict is
compared with the oracle's."""
import ctypes
import hashlib
import struct
import threading
import time

import numpy as np
import pytest

from test_table_repair import _engine, hooklib  # noqa: F401 (hooklib: the -DHS_TEST_HOOKS build, a fixture)

pytestmark = pytest.mark.gpu
K = 256
F_PARSE_OK, F_EQ, F_SMALL, F_STRICT = 1, 4, 8, 16
WHY_R_SMALL = 16
AUDIT_SIGCACHE = 32
HS_ERR_ARG = 2
FLAGS = 128  # hs_test_poke_sig's offset of the flag byte
L_ORDER = 2**252 + 27742317777372353535851937790883648493
ENTRIES = 1 << 14  # 4,096 buckets
BUCKETS = ENTRIES // 4
IDENTITY = (1).to_bytes(32, "little")


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(9100)
    seeds = rng.integers(0, 256, size=(K, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture(scope="module")
def eng(hooklib, keys):
    hooklib.hs_test_poke_sig.restype = ctypes.c_int
    hooklib.hs_test_poke_sig.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint8]
    e = _engine(hooklib, base_window=12, key_window=8)  # small comb tables: the session's engine holds its own on the same device
    assert e.committee_register(np.unique(keys[1], axis=0)).all()
    yield e
    e.close()


@pytest.fixture()
def q(eng):
    q = eng.queue(ring_records=4096)
    q.sig_cache(ENTRIES)
    yield q
    q.close()


def poke(eng, q, rec, offset, mask):
    assert eng.lib.hs_test_poke_sig(q.h, bytes(rec), offset, mask) == 0, eng.last_error


def digest(pre):
    return np.frombuffer(hashlib.sha512(pre).digest()[:32], np.uint8)


def signed(oracle, keys, kidx, digests):
    seeds, pks = keys
    kidx = np.asarray(kidx, np.uint32)
    d = np.ascontiguousarray(digests, np.uint8).reshape(-1, 32)
    sig = oracle.sign_batch(seeds, pks, kidx, d.reshape(-1), np.arange(len(kidx) + 1, dtype=np.uint64) * 32)
    return np.concatenate([sig, pks[kidx], d], axis=1)


def torsion_record(oracle, keys, k, msg):
    """R = the identity, S = k a: [S]B - [k]A = R holds without the cofactor, so batch-eq accepts it and strict rejects it (R is small):
    flags PARSE_OK | EQ | SMALL = 0x0d, why = HS_WHY_R_SMALL."""
    seed, pk = keys[0][k].tobytes(), keys[1][k].tobytes()
    h = hashlib.sha512(seed).digest()
    a = int.from_bytes(bytes([h[0] & 248]) + h[1:31] + bytes([(h[31] & 127) | 64]), "little")
    kk = int.from_bytes(hashlib.sha512(IDENTITY + pk + bytes(msg)).digest(), "little") % L_ORDER
    return np.frombuffer(IDENTITY + (kk * a % L_ORDER).to_bytes(32, "little") + pk + bytes(msg), np.uint8).copy()


def submit(q, recs, mode=0):
    """Records through the queue, at most 64 a request; verdicts in order."""
    recs = np.ascontiguousarray(recs, np.uint8).reshape(-1, 128)
    tickets = []
    for i in range(0, len(recs), 64):
        while (t := q.submit(recs[i:i + 64], mode)) is None:
            time.sleep(0.0005)
        tickets.append(t)
    return np.concatenate([q.wait(t) for t in tickets])


def oracle_bits(oracle, recs, mode=0):
    return oracle.verify_rec128(np.ascontiguousarray(recs, np.uint8).reshape(-1, 128), mode=mode).astype(bool)


def timeouts(oracle, keys, n, rng, rnd):
    """n Timeout author records of round rnd: author a[i] strict over SHA-512(round || high_qc_round[i])[..32]."""
    authors = rng.permutation(K)[:n]
    hq = rnd - 1 - rng.integers(0, 5, n)
    recs = signed(oracle, keys, authors, np.array([digest(struct.pack("<QQ", rnd, int(h))) for h in hq]))
    return recs, hq.astype(np.uint64)


def tc(eng, rnd, recs, hq):
    ok, votes = eng.verify_tcs(np.array([rnd], np.uint64), recs[:, :64], hq, tc_idx=np.zeros(len(recs), np.uint32), pk=recs[:, 64:96],
                               want_votes=True)
    return bool(ok[0]), votes


def wait_until(pred, timeout=20.0):
    deadline = time.time() + timeout
    while not pred():
        assert time.time() < deadline, "timed out"
        time.sleep(0.002)


def audit_ok(r, corrected):
    assert r["corrected"] == corrected, r
    if not corrected:
        assert r["first_position"] is None and r["first_stored"] == r["first_derived"] == r["first_why"] == 0


# ---------------------------------------------------------------------------------------------------------------- clean cache
def test_clean_cache_corrects_nothing(eng, q, oracle, keys):
    rng = np.random.default_rng(1)
    recs, hq = timeouts(oracle, keys, 200, rng, 1 << 30)
    recs[7, 40] ^= 1  # a rejected Timeout is not cached
    want = oracle_bits(oracle, recs)
    assert (submit(q, recs) == want).all()
    while (t := q.submit_group(recs)) is None:  # the TC: its votes are hits
        time.sleep(0.0005)
    assert (q.wait(t) == want).all()
    s = q.sig_stats()
    assert s["hits"] >= want.sum() and s["entries_held"] == want.sum()
    a0 = q.sig_audit_stats()
    r = q.sig_audit()
    audit_ok(r, 0)
    assert r["held"] == s["entries_held"] and r["skipped"] == 0
    assert q.sig_audit_stats() == dict(audits=a0["audits"] + 1, checked=a0["checked"] + r["held"], corrected=a0["corrected"],
                                       skipped=a0["skipped"], passes=a0["passes"] + 1)
    assert (submit(q, recs) == want).all()


# ---------------------------------------------------------------------------------------------------------------- false accept
def test_false_accept_is_corrected(eng, q, oracle, keys):
    rng = np.random.default_rng(2)
    rnd = 1 << 31
    votes, hq = timeouts(oracle, keys, 99, rng, rnd)
    hq_t = rnd - 1
    t = torsion_record(oracle, keys, int(rng.integers(0, K)), digest(struct.pack("<QQ", rnd, hq_t)))
    recs, hqs = np.concatenate([votes, t[None]]), np.concatenate([hq, [hq_t]]).astype(np.uint64)
    assert oracle_bits(oracle, t, 1)[0] and not oracle_bits(oracle, t, 0)[0]
    assert submit(q, t, 1)[0] and not submit(q, t, 0)[0]  # verified under batch-eq: cached with flags 0x0d
    q.sig_share(True)
    assert (submit(q, votes) == oracle_bits(oracle, votes)).all()
    ok, bits = tc(eng, rnd, recs, hqs)
    assert not ok and (bits == oracle_bits(oracle, recs)).all() and not bits[-1]
    poke(eng, q, t, FLAGS, F_STRICT)  # the entry now says strict-valid
    # the poke bites: the record is strict-accepted through the queue and through the shared hs_verify_tcs
    assert submit(q, t, 0)[0]
    ok, bits = tc(eng, rnd, recs, hqs)
    assert ok and bits[-1]
    r = q.sig_audit()
    audit_ok(r, 1)
    assert (r["first_stored"], r["first_derived"], r["first_why"]) == (F_PARSE_OK | F_EQ | F_SMALL | F_STRICT, F_PARSE_OK | F_EQ | F_SMALL,
                                                                       WHY_R_SMALL)
    assert not submit(q, t, 0)[0] and submit(q, t, 1)[0]
    ok, bits = tc(eng, rnd, recs, hqs)
    assert not ok and (bits == oracle_bits(oracle, recs)).all()
    audit_ok(q.sig_audit(), 0)


# ---------------------------------------------------------------------------------------------------------------- false reject
def test_false_reject_is_corrected(eng, q, oracle, keys):
    rng = np.random.default_rng(3)
    recs = signed(oracle, keys, rng.integers(0, K, 8), rng.integers(0, 256, (8, 32), dtype=np.uint8))
    assert submit(q, recs).all()
    v = recs[3]
    poke(eng, q, v, FLAGS, F_STRICT)  # flags 0x05: the honest record is rejected from the cache
    assert not submit(q, v, 0)[0] and submit(q, v, 1)[0]
    q.explain(64, 1 << 16)
    while (t := q.submit_explain(v[None])) is None:
        time.sleep(0.0005)
    assert q.wait(t)[0] == 0  # the table-free re-check calls it valid: an engine fault
    r = q.sig_audit()
    audit_ok(r, 1)
    assert (r["first_stored"], r["first_derived"], r["first_why"]) == (F_PARSE_OK | F_EQ, F_PARSE_OK | F_EQ | F_STRICT, 0)
    assert (submit(q, recs) == oracle_bits(oracle, recs)).all()


# ---------------------------------------------------------------------------------------------------------------- word poke
@pytest.mark.parametrize("offset", [5, 40, 70, 100])  # a byte of R, S, A and the Digest
def test_word_poke_gets_the_recheck_of_the_new_bytes(eng, q, oracle, keys, offset):
    rng = np.random.default_rng(4 + offset)
    recs = signed(oracle, keys, rng.integers(0, K, 4), rng.integers(0, 256, (4, 32), dtype=np.uint8))
    assert submit(q, recs).all()
    v = recs[1]
    poke(eng, q, v, offset, 0x04)
    w = v.copy()
    w[offset] ^= 0x04
    why = int(eng.explain(w[None])[0])
    want = (0 if why & 3 else F_PARSE_OK) | (0 if why & ~24 else F_EQ) | (F_SMALL if why & 24 else 0) | (0 if why else F_STRICT)
    assert want != F_PARSE_OK | F_EQ | F_STRICT and not oracle_bits(oracle, w, 0)[0]
    r = q.sig_audit()
    audit_ok(r, 1)
    assert (r["first_stored"], r["first_derived"], r["first_why"]) == (F_PARSE_OK | F_EQ | F_STRICT, want, why)
    audit_ok(q.sig_audit(), 0)
    # the original record misses (its entry now holds other bytes) and verifies as the oracle does, and so do the new bytes
    h0 = q.sig_stats()["hits"]
    assert submit(q, v, 0)[0] and q.sig_stats()["hits"] == h0
    assert submit(q, w, 0)[0] == oracle_bits(oracle, w, 0)[0] and submit(q, w, 1)[0] == oracle_bits(oracle, w, 1)[0]


# ---------------------------------------------------------------------------------------------------------------- slices and errors
def test_slices_find_what_the_whole_table_finds(eng, q, oracle, keys):
    rng = np.random.default_rng(5)
    recs = signed(oracle, keys, rng.integers(0, K, 600), rng.integers(0, 256, (600, 32), dtype=np.uint8))
    assert submit(q, recs).all()
    bad = rng.choice(600, 12, replace=False)

    def corrupt():
        for i in bad:
            poke(eng, q, recs[i], FLAGS, F_STRICT)

    corrupt()
    parts = [q.sig_audit(b, n) for b, n in ((0, 1), (1, 1000), (1001, 95), (1096, 0))]
    corrupt()
    whole = q.sig_audit(0, 0)
    assert sum(p["held"] for p in parts) == whole["held"] == q.sig_stats()["entries_held"]
    assert sum(p["corrected"] for p in parts) == whole["corrected"] == 12
    firsts = [p["first_position"] for p in parts if p["first_position"] is not None]
    assert min(firsts) == whole["first_position"] and whole["first_stored"] == F_PARSE_OK | F_EQ
    audit_ok(q.sig_audit(), 0)
    assert (submit(q, recs) == True).all()  # noqa: E712
    # bad ranges and a cache that is off: HS_ERR_ARG, out untouched
    out = (ctypes.c_uint64 * 7)(*([0xabcd] * 7))
    for first, n in ((BUCKETS, 0), (BUCKETS - 1, 2), (0, BUCKETS + 1), (2**40, 1)):
        assert eng.lib.hs_queue_sig_audit(q.h, first, n, out) == HS_ERR_ARG and list(out) == [0xabcd] * 7, (first, n)
    a0 = q.sig_audit_stats()
    q.sig_cache(0)
    assert eng.lib.hs_queue_sig_audit(q.h, 0, 0, out) == HS_ERR_ARG and list(out) == [0xabcd] * 7
    assert q.sig_audit_stats() == a0


# ---------------------------------------------------------------------------------------------------------------- concurrency
def test_audit_beside_a_vote_burst_changes_no_verdict(eng, q, oracle, keys):
    rng = np.random.default_rng(6)
    recs = signed(oracle, keys, rng.integers(0, K, 667), rng.integers(0, 256, (667, 32), dtype=np.uint8))
    recs[rng.choice(667, 30, replace=False), 40] ^= 2
    want = oracle_bits(oracle, recs)
    assert (submit(q, recs) == want).all()  # the burst's records are in the table
    results, stop = [], threading.Event()

    def audits():
        while not stop.is_set():
            results.append(q.sig_audit())

    th = threading.Thread(target=audits)
    th.start()
    try:
        for _ in range(3):
            assert (submit(q, recs) == want).all()
    finally:
        stop.set()
        th.join()
    assert results and all(r["corrected"] == 0 for r in results), results[:3]
    # a resize waits for the audit in flight, then serves the new, empty table
    done = []
    th = threading.Thread(target=lambda: done.append(q.sig_audit()))
    th.start()
    q.sig_cache(ENTRIES * 2)
    th.join()
    assert len(done) == 1 and done[0]["corrected"] == 0
    r = q.sig_audit()
    assert r["held"] == 0 and q.sig_stats()["entries_held"] == 0
    assert (submit(q, recs) == want).all()
    assert q.sig_audit()["held"] == want.sum()


# ---------------------------------------------------------------------------------------------------------------- scrub
def test_scrub_corrects_within_a_pass(eng, oracle, keys):
    rng = np.random.default_rng(7)
    recs = signed(oracle, keys, rng.integers(0, K, 64), rng.integers(0, 256, (64, 32), dtype=np.uint8))
    order = np.unique(keys[1], axis=0)
    per_tick, period_us = 512, 2000
    limit = -(-BUCKETS // per_tick) + 1  # a pass of slices, and the tick in progress when the entry was poked
    seen = []

    def ticks():
        s = eng.scrub_stats()
        return s["ticks"] + s["ticks_paused"]

    def wait_ticks(n):
        t = ticks()
        wait_until(lambda: ticks() >= t + n)

    q = eng.queue()
    try:
        q.sig_cache(ENTRIES)
        assert submit(q, recs).all()
        eng.scrub_sig_cache(q, per_tick)
        eng.scrub_start(order, period_us=period_us, slots_per_tick=K, base_entries_per_tick=1 << 20,
                        callback=lambda found, failed, first_slot: seen.append((found, failed, first_slot, ticks())))
        try:
            wait_ticks(1)
            a0 = q.sig_audit_stats()
            poke(eng, q, recs[9], FLAGS, F_STRICT)
            t0 = ticks()
            wait_until(lambda: seen)
            assert seen[0][:3] == (AUDIT_SIGCACHE, 0, 2**64 - 1) and seen[0][3] - t0 <= limit, (seen, t0)
            assert (submit(q, recs) == True).all()  # noqa: E712
            a1 = q.sig_audit_stats()
            assert a1["corrected"] == a0["corrected"] + 1 and a1["audits"] > a0["audits"]
            wait_until(lambda: q.sig_audit_stats()["passes"] > a0["passes"])
            # detached: a poke stays until an audit is asked for
            eng.scrub_sig_cache(None)
            wait_ticks(1)
            n0 = q.sig_audit_stats()["audits"]
            poke(eng, q, recs[10], FLAGS, F_STRICT)
            wait_ticks(2 * limit)
            assert q.sig_audit_stats()["audits"] == n0 and not submit(q, recs[10])[0]
            audit_ok(q.sig_audit(), 1)
            # attached again, then the queue destroyed under the running scrub
            eng.scrub_sig_cache(q, per_tick)
            wait_ticks(3)
        finally:
            q.close()
        wait_ticks(5)
    finally:
        eng.scrub_stop()
    assert len(seen) == 1, seen
