"""The host-pointer entry points: hs_verify_rec128, hs_verify_var, hs_verify_batch_shared_msg, hs_verify_committee, hs_verify_qcs,
hs_verify_tcs, hs_verify_groups, hs_keygen_batch, hs_sign_digests, hs_digest32_batch and hs_verify_msgs.  On each path of each call:
the kernel launches of one call, and outputs bit-equal to the oracle at n = 1, 31, 32, 33 and 2,500, with null optional inputs and
outputs, and byte totals that are not a multiple of 8.  An out-of-range index in hs_verify_qcs, hs_verify_tcs or hs_verify_groups is
HS_ERR_ARG and leaves the caller's output bitmaps as they were."""
import hashlib

import numpy as np
import pytest

from test_groups_dev import FOREIGN, K, _clear, _register, expected, keys, make_burst, run_host  # noqa: F401 (keys is a fixture)

pytestmark = pytest.mark.gpu
SIZES = (1, 31, 32, 33, 2500)
HS_ERR_ARG = 2


@pytest.fixture
def committee(engine, keys):
    """The first K keys registered in order (committee index = key index); cleared afterwards."""
    _register(engine, keys)
    yield
    _clear(engine)


def launches(engine, call):
    """(what call() returns, the kernel launches it made)"""
    l0 = engine.kernel_launches
    out = call()
    return out, engine.kernel_launches - l0


def sign(oracle, keys, kidx, msgs32):
    seeds, pks = keys
    return oracle.sign_batch(seeds, pks, kidx, msgs32.reshape(-1), np.arange(len(kidx) + 1, dtype=np.uint64) * 32)


def flip_bits(rng, a, frac, cols):
    """One flipped bit in about `frac` of the rows of `a`, in a byte among `cols`."""
    for i in np.flatnonzero(rng.random(a.shape[0]) < frac):
        a[i, int(rng.choice(cols))] ^= np.uint8(1 << int(rng.integers(8)))


def records(oracle, keys, rng, n, foreign=0):
    """n (sig | pk | msg) records signed by committee keys (the last `foreign` by keys outside it), about 10 % of them with a flipped
    bit in the signature or the message (the key bytes stay registered)."""
    kidx = rng.integers(0, K, n).astype(np.uint32)
    if foreign:
        kidx[-foreign:] = K + rng.integers(0, FOREIGN, foreign)
    msgs = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    recs = np.concatenate([sign(oracle, keys, kidx, msgs), keys[1][kidx], msgs], axis=1)
    flip_bits(rng, recs, 0.1, np.r_[0:64, 96:128])
    return recs, kidx


def offsets(lens):
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    return off


def ragged(rng, n, hi):
    """n message lengths in [0, hi) whose total is not a multiple of 8."""
    lens = rng.integers(0, hi, n)
    if lens.sum() % 8 == 0:
        lens[0] += 1
    return lens


# ---- the verify calls over records
@pytest.mark.parametrize("n", SIZES)
def test_verify_rec128(engine, oracle, keys, committee, n):
    """n <= 64 with every key registered: one latency-path launch.  Otherwise (n = 2,500, or a key outside the committee): lookup, miss
    pass, main and finish."""
    rng = np.random.default_rng(n)
    for foreign in ((0, 1) if n <= 64 else (3,)):
        recs, _ = records(oracle, keys, rng, n, foreign)
        for mode in (0, 1):
            got, dl = launches(engine, lambda: engine.verify_rec128(recs, mode=mode))
            assert dl == (1 if n <= 64 and not foreign else 4), (foreign, mode)
            assert (got == oracle.verify_rec128(recs, mode=mode)).all(), (foreign, mode)


@pytest.mark.parametrize("n", SIZES)
def test_verify_var(engine, oracle, keys, committee, n):
    """Messages of 0 to 299 bytes whose total is not a multiple of 8: lookup, miss pass, main and finish."""
    rng = np.random.default_rng(10 + n)
    seeds, pks = keys
    off = offsets(ragged(rng, n, 300))
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    kidx = rng.integers(0, K + FOREIGN, n).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, kidx, msgs, off)
    flip_bits(rng, sig, 0.1, np.arange(64))
    for mode in (0, 1):
        got, dl = launches(engine, lambda: engine.verify_var(sig, pks[kidx], msgs, off, mode=mode))
        assert dl == 4 and (got == oracle.verify_var(sig, pks[kidx], msgs, off, mode=mode)).all(), mode


@pytest.mark.parametrize("n", SIZES)
def test_verify_batch_shared_msg(engine, oracle, keys, committee, n):
    """Votes over one digest, all valid and then with bad votes, with and without the bitmap: one latency-path launch for n <= 64,
    lookup, miss pass, main and finish for n = 2,500."""
    rng = np.random.default_rng(20 + n)
    digest = rng.integers(0, 256, 32, dtype=np.uint8)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    votes = np.concatenate([keys[1][kidx], sign(oracle, keys, kidx, np.tile(digest, (n, 1)))], axis=1)
    bad = votes.copy()
    bad[-1, 40] ^= 1
    flip_bits(rng, bad, 0.1, np.arange(32, 96))
    for v, valid in ((votes, True), (bad, False)):
        want_ok, want_bits = oracle.verify_batch_shared_msg(digest, v)
        assert want_ok == valid
        (ok, bits), dl = launches(engine, lambda: engine.verify_batch_shared_msg(digest, v, want_bitmap=True))
        assert dl == (1 if n <= 64 else 4) and ok == want_ok and (bits == want_bits).all(), valid
        ok, dl = launches(engine, lambda: engine.verify_batch_shared_msg(digest, v))
        assert dl == (1 if n <= 64 else 4) and ok == want_ok, valid


@pytest.mark.parametrize("n", SIZES)
def test_verify_committee(engine, oracle, keys, committee, n):
    """Indices with msg_idx and with msg_idx == NULL (one digest), one index outside the committee: one latency-path launch for n <= 64,
    main and finish for n = 2,500."""
    rng = np.random.default_rng(30 + n)
    pks = keys[1]
    for with_midx in (True, False):
        digests = rng.integers(0, 256, (max(1, n // 3) if with_midx else 1, 32), dtype=np.uint8)
        midx = rng.integers(0, digests.shape[0], n).astype(np.uint32) if with_midx else np.zeros(n, np.uint32)
        vidx = rng.integers(0, K, n).astype(np.uint32)
        sig = sign(oracle, keys, vidx, digests[midx])
        flip_bits(rng, sig, 0.1, np.arange(64))
        vidx[n // 2] = K + 5  # not a committee index: rejected
        want = oracle.verify_rec128(np.concatenate([sig, pks[np.minimum(vidx, K - 1)], digests[midx]], axis=1))
        want[n // 2] = False
        for mode in (0, 1):
            got, dl = launches(engine, lambda: engine.verify_committee(vidx, sig, digests, msg_idx=midx if with_midx else None, mode=mode))
            assert dl == (1 if n <= 64 else 2) and (got == want).all(), (with_midx, mode)


# ---- certificates
def qc_case(oracle, keys, rng, n):
    """n votes over n // 8 + 2 QCs (the last without votes): (preimages, sig, qc_idx, kidx, vote verdicts, QC verdicts)."""
    n_qc = n // 8 + 2
    pre = rng.integers(0, 256, (n_qc, 40), dtype=np.uint8)
    digests = np.array([np.frombuffer(hashlib.sha512(p.tobytes()).digest()[:32], np.uint8) for p in pre])
    qi = np.sort(rng.integers(0, n_qc - 1, n)).astype(np.uint32)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    sig = sign(oracle, keys, kidx, digests[qi])
    flip_bits(rng, sig, 0.05, np.arange(64))
    votes = oracle.verify_rec128(np.concatenate([sig, keys[1][kidx], digests[qi]], axis=1), mode=1)
    qcs = np.ones(n_qc, bool)
    np.logical_and.at(qcs, qi, votes)
    return pre, sig, qi, kidx, votes, qcs


@pytest.mark.parametrize("n", SIZES)
def test_verify_qcs(engine, oracle, keys, committee, n):
    """QC digest, then the verify pass (lookup, miss pass, main, finish with key bytes; main and finish with indices), then the QC AND."""
    rng = np.random.default_rng(40 + n)
    pre, sig, qi, kidx, want_v, want_q = qc_case(oracle, keys, rng, n)
    for by_index in (False, True):
        kw = dict(validator_idx=kidx) if by_index else dict(pk=keys[1][kidx])
        per_call = 4 if by_index else 6
        (q, v), dl = launches(engine, lambda: engine.verify_qcs(pre, sig, qi, want_votes=True, **kw))
        assert dl == per_call and (v == want_v).all() and (q == want_q).all(), by_index
        q, dl = launches(engine, lambda: engine.verify_qcs(pre, sig, qi, **kw))
        assert dl == per_call and (q == want_q).all() and q[-1], by_index


@pytest.mark.parametrize("n", SIZES)
def test_verify_tcs(engine, oracle, keys, committee, n):
    """TC digests, then the verify pass, then (with tc_idx) the TC AND; without tc_idx each vote is its own certificate."""
    rng = np.random.default_rng(50 + n)
    pks = keys[1]
    for with_idx in (True, False):
        n_tc = n // 8 + 2 if with_idx else n
        rounds = rng.integers(0, 1 << 63, n_tc, dtype=np.uint64)
        ti = np.sort(rng.integers(0, n_tc - 1, n)).astype(np.uint32) if with_idx else np.arange(n, dtype=np.uint32)
        hq = rng.integers(0, 1 << 63, n, dtype=np.uint64)
        digests = np.array([np.frombuffer(hashlib.sha512(rounds[t].astype("<u8").tobytes() + h.astype("<u8").tobytes()).digest()[:32], np.uint8)
                            for t, h in zip(ti, hq)])
        kidx = rng.integers(0, K, n).astype(np.uint32)
        sig = sign(oracle, keys, kidx, digests)
        flip_bits(rng, sig, 0.05, np.arange(64))
        want_v = oracle.verify_rec128(np.concatenate([sig, pks[kidx], digests], axis=1), mode=0)
        want_t = np.ones(n_tc, bool)
        np.logical_and.at(want_t, ti, want_v)
        for by_index in (False, True):
            kw = dict(validator_idx=kidx) if by_index else dict(pk=pks[kidx])
            per_call = (3 if by_index else 5) + (1 if with_idx else 0)
            for want_votes in (True, False):
                out, dl = launches(engine, lambda: engine.verify_tcs(rounds, sig, hq, tc_idx=ti if with_idx else None, want_votes=want_votes, **kw))
                t, v = out if want_votes else (out, want_v)
                assert dl == per_call and (t == want_t).all() and (v == want_v).all(), (with_idx, by_index, want_votes)


@pytest.mark.parametrize("n", SIZES)
def test_verify_groups(engine, oracle, keys, committee, n):
    """Digest, lookup, miss pass, main, finish and the group AND with key bytes; digest, main, finish and the AND with indices.  With and
    without modes and the item bitmap, over preimages whose total is not a multiple of 8."""
    rng = np.random.default_rng(60 + n)
    b = make_burst(oracle, keys, rng, n)
    if int(b["off"][-1]) % 8 == 0:  # one more byte in the last preimage, which no item may name
        b = dict(b, pre=np.append(b["pre"], np.uint8(7)), off=np.append(b["off"], b["off"][-1] + np.uint64(1)))
    assert int(b["off"][-1]) % 8
    for indexed in (False, True):
        for modes in (True, False):
            want_g, want_i = expected(oracle, keys, b, indexed, modes)
            (g, items), dl = launches(engine, lambda: run_host(engine, b, indexed, modes))
            assert dl == (4 if indexed else 6) and (g == want_g).all() and (items == want_i).all(), (indexed, modes)
            kw = dict(validator_idx=b["kidx"]) if indexed else dict(pk=b["pk"])
            g = engine.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"] if modes else None, **kw)
            assert (g == want_g).all(), (indexed, modes)


@pytest.mark.parametrize("n", SIZES)
def test_verify_groups_without_preimage_bytes(engine, oracle, keys, committee, n):
    """Every preimage empty: preimages == NULL and pre_off all zero.  Every item signs Digest("")."""
    rng = np.random.default_rng(70 + n)
    n_msgs, n_groups = 3, n // 4 + 2
    empty = np.frombuffer(hashlib.sha512(b"").digest()[:32], np.uint8)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    sig = sign(oracle, keys, kidx, np.tile(empty, (n, 1)))
    flip_bits(rng, sig, 0.1, np.arange(64))
    mi = rng.integers(0, n_msgs, n).astype(np.uint32)
    gi = np.sort(rng.integers(0, n_groups - 1, n)).astype(np.uint32)
    modes = rng.integers(0, 2, n).astype(np.uint8)
    recs = np.concatenate([sig, keys[1][kidx], np.tile(empty, (n, 1))], axis=1)
    want_i = np.where(modes == 1, oracle.verify_rec128(recs, mode=1), oracle.verify_rec128(recs, mode=0))
    want_g = np.ones(n_groups, bool)
    np.logical_and.at(want_g, gi, want_i)
    for indexed in (False, True):
        kw = dict(validator_idx=kidx) if indexed else dict(pk=keys[1][kidx])
        (g, items), dl = launches(engine, lambda: engine.verify_groups(np.zeros(0, np.uint8), np.zeros(n_msgs + 1, np.uint64), sig, mi, gi, n_groups,
                                                                      mode=modes, want_items=True, **kw))
        assert dl == (4 if indexed else 6) and (items == want_i).all() and (g == want_g).all() and g[-1], indexed


# ---- load generation and digests
@pytest.mark.parametrize("n", SIZES)
def test_keygen_and_sign(engine, oracle, keys, n):
    """One launch each; signing with key_idx and with key_idx == NULL (signature i by key i)."""
    rng = np.random.default_rng(80 + n)
    seeds = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    pks, dl = launches(engine, lambda: engine.keygen_batch(seeds))
    assert dl == 1 and (pks == oracle.keygen_batch(seeds)).all()
    digests = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    for ki in (rng.integers(0, n, n).astype(np.uint32), None):
        sig, dl = launches(engine, lambda: engine.sign_digests(seeds, pks, digests, key_idx=ki))
        kk = np.arange(n, dtype=np.uint32) if ki is None else ki
        assert dl == 1 and (sig == oracle.sign_batch(seeds, pks, kk, digests.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)).all()


@pytest.mark.parametrize("n", SIZES)
def test_digest32_batch(engine, oracle, n):
    """One launch: the generic kernel for short messages, the long-message kernel for up to 64 messages of 1,024 bytes or more on average;
    totals that are not a multiple of 8."""
    rng = np.random.default_rng(90 + n)
    for hi in ((300, 3000) if n <= 64 else (300,)):
        lens = ragged(rng, n, hi)
        if hi > 300:
            lens[0] += 1024 * n  # at least 1,024 bytes per message on average
            assert lens.sum() % 8
        off = offsets(lens)
        data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
        got, dl = launches(engine, lambda: engine.digest32_batch(data, off))
        assert dl == 1 and (got == oracle.digest32_batch(data, off)).all(), hi


# ---- the end-to-end call
@pytest.mark.parametrize("n", SIZES)
def test_verify_msgs(engine, oracle, keys, committee, n):
    """Per chunk: the digest, then lookup, miss pass, main and finish with key bytes, or main and finish with indices.  512-byte messages
    take the fixed-length digest kernel, 100-byte ones the generic one."""
    rng = np.random.default_rng(100 + n)
    pks = keys[1]
    for L in (512, 100):
        msgs = rng.integers(0, 256, (n, L), dtype=np.uint8)
        d = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
        kidx = rng.integers(0, K, n).astype(np.uint32)
        sig = sign(oracle, keys, kidx, d)
        flip_bits(rng, sig, 0.1, np.arange(64))
        want = oracle.verify_rec128(np.concatenate([sig, pks[kidx], d], axis=1))
        for kw, per_chunk in ((dict(pk=pks[kidx]), 5), (dict(validator_idx=kidx), 3)):
            got, dl = launches(engine, lambda: engine.verify_msgs(sig, msgs.reshape(-1), L, **kw))
            assert dl == per_chunk and (got == want).all(), (L, per_chunk)


def test_verify_msgs_chunk_pipeline(engine, oracle, keys, committee, monkeypatch):
    """HS_CHUNK_RECORDS=1024: 2,500 records in three chunks over the two staging buffers, the third reusing the first's."""
    monkeypatch.setenv("HS_CHUNK_RECORDS", "1024")
    rng = np.random.default_rng(111)
    n, L, pks = 2500, 144, keys[1]
    msgs = rng.integers(0, 256, (n, L), dtype=np.uint8)
    d = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
    kidx = rng.integers(0, K + FOREIGN, n).astype(np.uint32)
    sig = sign(oracle, keys, kidx, d)
    flip_bits(rng, sig, 0.1, np.arange(64))
    want = oracle.verify_rec128(np.concatenate([sig, pks[kidx], d], axis=1))
    got, dl = launches(engine, lambda: engine.verify_msgs(sig, msgs.reshape(-1), L, pk=pks[kidx]))
    assert dl == 3 * 5 and (got == want).all()


def test_certificates_without_votes_are_accepted(engine):
    """No votes or items: every certificate and group is accepted, and no kernel runs."""
    none64 = np.zeros((0, 64), np.uint8)
    q, dl = launches(engine, lambda: engine.verify_qcs(np.zeros((33, 40), np.uint8), none64, np.zeros(0, np.uint32), pk=np.zeros((0, 32), np.uint8)))
    assert dl == 0 and q.shape == (33,) and q.all()
    t, dl = launches(engine, lambda: engine.verify_tcs(np.zeros(33, np.uint64), none64, np.zeros(0, np.uint64), tc_idx=np.zeros(0, np.uint32),
                                                       validator_idx=np.zeros(0, np.uint32)))
    assert dl == 0 and t.shape == (33,) and t.all()
    g, dl = launches(engine, lambda: engine.verify_groups(np.zeros(0, np.uint8), np.zeros(1, np.uint64), none64, np.zeros(0, np.uint32),
                                                          np.zeros(0, np.uint32), 33, pk=np.zeros((0, 32), np.uint8)))
    assert dl == 0 and g.shape == (33,) and g.all()


# ---- argument errors
@pytest.mark.parametrize("case", ["qc_idx", "tc_idx", "msg_idx", "group_idx", "mode", "qcs_indexed", "tcs_indexed", "groups_indexed"])
def test_argument_errors_leave_outputs_untouched(engine, case):
    """An index out of range, a mode byte above 1, or validator indices without a registered committee: HS_ERR_ARG, and the zeroed
    output bitmaps stay zeroed, so no certificate is reported accepted."""
    lib, h, p = engine.lib, engine.h, lambda a: None if a is None else a.ctypes.data
    n, n_cert = 40, 5
    sig = np.zeros((n, 64), np.uint8)
    pk, vidx = (None, np.zeros(n, np.uint32)) if case.endswith("indexed") else (np.zeros((n, 32), np.uint8), None)
    idx = (np.arange(n) % n_cert).astype(np.uint32)
    bad = idx.copy()
    bad[17] = n_cert
    mi, mode = np.zeros(n, np.uint32), np.zeros(n, np.uint8)
    if case == "msg_idx":
        mi[17] = 2
    elif case == "mode":
        mode[17] = 2
    out_items, out_certs = np.zeros((n + 31) // 32, np.uint32), np.zeros((n_cert + 31) // 32, np.uint32)
    _clear(engine)
    if case.startswith("qc"):
        rc = lib.hs_verify_qcs(h, p(np.zeros((n_cert, 40), np.uint8)), n_cert, p(pk), p(vidx), p(sig), p(bad if case == "qc_idx" else idx), n,
                               p(out_items), p(out_certs))
    elif case.startswith("tc"):
        rc = lib.hs_verify_tcs(h, p(np.zeros(n_cert, np.uint64)), n_cert, p(pk), p(vidx), p(sig), p(np.zeros(n, np.uint64)),
                               p(bad if case == "tc_idx" else idx), n, p(out_items), p(out_certs))
    else:
        rc = lib.hs_verify_groups(h, p(np.zeros(48, np.uint8)), p(np.array([0, 16, 48], np.uint64)), 2, p(sig), p(pk), p(vidx), p(mi),
                                  p(bad if case == "group_idx" else idx), p(mode), n, n_cert, p(out_items), p(out_certs))
    assert rc == HS_ERR_ARG
    assert (b"without a registered committee" if case.endswith("indexed") else b"out of range") in lib.hs_last_error(h)
    assert not out_items.any() and not out_certs.any()
