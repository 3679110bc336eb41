"""GPU parity: the CUDA path (through the C ABI of include/hs_crypto.h) against the CPU oracle and the committed golden
fixtures.  Bit-exact: every verdict bit must equal the oracle's."""
import hashlib

import numpy as np
import pytest

from oracle_api import EQ_OK, STRICT, make_workload, to_rec128

pytestmark = pytest.mark.gpu


def _golden_arrays(golden, only32=False):
    vs = [v for v in golden["vectors"] if (len(v["msg"]) == 64 or not only32)]
    sig = np.array([np.frombuffer(bytes.fromhex(v["sig"]), np.uint8) for v in vs])
    pk = np.array([np.frombuffer(bytes.fromhex(v["pk"]), np.uint8) for v in vs])
    msgs = [bytes.fromhex(v["msg"]) for v in vs]
    return vs, sig, pk, msgs


def test_golden_vectors_rec128_strict_and_batch_eq(engine, golden):
    vs, sig, pk, msgs = _golden_arrays(golden, only32=True)
    recs = np.concatenate([sig, pk, np.array([np.frombuffer(m, np.uint8) for m in msgs])], axis=1)
    got_s = engine.verify_rec128(recs, mode=0)
    got_e = engine.verify_rec128(recs, mode=1)
    for v, a, b in zip(vs, got_s, got_e):
        assert bool(a) == v["strict"], v["name"]
        assert bool(b) == v["batch_eq"], v["name"]


def test_golden_vectors_variable_length(engine, golden):
    vs, sig, pk, msgs = _golden_arrays(golden)
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    got = engine.verify_var(sig, pk, np.frombuffer(b"".join(msgs), np.uint8), off, mode=0)
    for v, a in zip(vs, got):
        assert bool(a) == v["strict"], v["name"]
    got = engine.verify_var(sig, pk, np.frombuffer(b"".join(msgs), np.uint8), off, mode=1)
    for v, a in zip(vs, got):
        assert bool(a) == v["batch_eq"], v["name"]


def test_golden_vectors_committee(engine, oracle, golden):
    vs, sig, pk, msgs = _golden_arrays(golden, only32=True)
    keys, inv = np.unique(pk, axis=0, return_inverse=True)
    valid = engine.committee_register(keys)
    digests = np.array([np.frombuffer(m, np.uint8) for m in msgs])
    for mode, field in ((0, "strict"), (1, "batch_eq")):
        got = engine.verify_committee(inv.astype(np.uint32), sig, digests, msg_idx=np.arange(len(vs), dtype=np.uint32), mode=mode)
        for v, a in zip(vs, got):
            assert bool(a) == v[field], (v["name"], field)
    for k, ok in zip(keys, valid):   # out_valid_bitmap = "the key decompresses" (PublicKey::from_bytes succeeds)
        assert bool(ok) == oracle.decompress_ok(k.tobytes()), k.tobytes().hex()
    # unknown authority index -> reject
    got = engine.verify_committee(np.array([len(keys) + 5], dtype=np.uint32), sig[:1], digests[:1])
    assert not got[0]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 128, 129, 1000])
def test_ragged_sizes(engine, oracle, n):
    w = make_workload(oracle, n, n_keys=5, seed=100 + n, corrupt_frac=0.2)
    recs = to_rec128(w)
    got = engine.verify_rec128(recs)
    want = oracle.verify_rec128(recs)
    assert (got == want).all()
    assert got[~w["corrupted"]].all()


def test_empty_inputs(engine):
    assert engine.verify_rec128(np.zeros((0, 128), np.uint8)).shape == (0,)
    assert engine.verify_batch_shared_msg(bytes(32), np.zeros((0, 96), np.uint8)) is True  # dalek verify_batch(&[]) is Ok
    assert engine.digest32_batch(b"", np.zeros(1, np.uint64)).shape == (0, 32)


def test_random_parity_rec128_with_corruptions(engine, oracle):
    """16 Ki records, 1,024 keys, 3 % single-bit corruptions over sig|pk|msg: every bit equals the oracle's."""
    w = make_workload(oracle, 1 << 14, n_keys=1024, seed=7, corrupt_frac=0.03)
    recs = to_rec128(w)
    for mode in (0, 1):
        got = engine.verify_rec128(recs, mode=mode)
        want = oracle.verify_rec128(recs, mode=mode)
        assert (got == want).all(), np.nonzero(got != want)[0][:10]
    assert (~want).sum() >= 400


def test_variable_length_messages_parity(engine, oracle):
    rng = np.random.default_rng(9)
    n = 600
    lens = rng.integers(0, 700, n)
    lens[:8] = [0, 1, 47, 48, 111, 112, 175, 176]
    seeds = rng.integers(0, 256, (16, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    kidx = (np.arange(n) % 16).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, kidx, msgs, off)
    pk = pks[kidx].copy()
    for i in range(0, n, 7):
        sig[i, int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
    got = engine.verify_var(sig, pk, msgs, off)
    want = oracle.verify_var(sig, pk, msgs, off)
    assert (got == want).all()
    assert want.sum() > n // 2 and (~want).sum() > 50


def test_512_byte_messages_config2_shape(engine, oracle):
    """BASELINE config 2 shape at a size the oracle finishes quickly: 512 B messages, 1 % seeded corruptions;
    variant B (raw PureEdDSA over 512 B) and variant A (Digest(msg) on the GPU, then verify over the digest)."""
    n = 4096
    w = make_workload(oracle, n, n_keys=256, msg_len=512, seed=21, corrupt_frac=0.01)
    got = engine.verify_var(w["sig"], w["pk"], w["msgs"], w["off"])
    want = oracle.verify_var(w["sig"], w["pk"], w["msgs"], w["off"])
    assert (got == want).all() and (~want).sum() >= 30
    # variant A
    d_gpu = engine.digest32_batch(w["msgs"], w["off"])
    d_cpu = oracle.digest32_batch(w["msgs"].tobytes(), w["off"])
    assert (d_gpu == d_cpu).all()
    kidx = w["key_idx"]
    sig = oracle.sign_batch(w["seeds"], w["pks"], kidx, d_cpu.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    recs = np.concatenate([sig, w["pks"][kidx], d_gpu], axis=1)
    assert engine.verify_rec128(recs).all()


def test_shared_message_votes(engine, oracle):
    """Signature::verify_batch shape (QC::verify, consensus/src/messages.rs:197): committee 1,000 -> quorum 667."""
    n = 667
    rng = np.random.default_rng(12)
    seeds = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    digest = oracle.digest32(bytes(32) + (7).to_bytes(8, "little"))
    msgs = np.tile(np.frombuffer(digest, np.uint8), n)
    sig = oracle.sign_batch(seeds, pks, np.arange(n, dtype=np.uint32), msgs, np.arange(n + 1, dtype=np.uint64) * 32)
    votes = np.concatenate([pks, sig], axis=1)
    ok, bits = engine.verify_batch_shared_msg(digest, votes, want_bitmap=True)
    assert ok and bits.all()
    assert engine.verify_batch_shared_msg(digest, votes) is True
    votes[401, 50] ^= 0x20
    ok, bits = engine.verify_batch_shared_msg(digest, votes, want_bitmap=True)
    ok_o, bits_o = oracle.verify_batch_shared_msg(digest, votes, nthreads=8)
    assert ok == ok_o is False and (bits == bits_o).all() and not bits[401]


def test_committee_mode_parity(engine, oracle):
    """Committee of 200 validators, 40 QC digests, 8,000 votes, 2 % corrupted; indexed mode == generic mode == oracle."""
    rng = np.random.default_rng(33)
    N, Q, n = 200, 40, 8000
    seeds = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    digests = np.array([np.frombuffer(oracle.digest32(rng.bytes(32) + int(r).to_bytes(8, "little")), np.uint8) for r in range(Q)])
    vidx = rng.integers(0, N, n).astype(np.uint32)
    midx = rng.integers(0, Q, n).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, vidx, digests[midx].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    bad = rng.choice(n, n // 50, replace=False)
    for i in bad:
        sig[i, int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
    assert engine.committee_register(pks).all()
    got = engine.verify_committee(vidx, sig, digests, msg_idx=midx)
    recs = np.concatenate([sig, pks[vidx], digests[midx]], axis=1)
    want = oracle.verify_rec128(recs)
    assert (got == want).all()
    assert (engine.verify_rec128(recs) == want).all()
    assert (~want).sum() >= len(bad) - 2


def test_digest32_batch_parity(engine, oracle, golden):
    rng = np.random.default_rng(44)
    lens = list(range(0, 270)) + [511, 512, 513, 4096, 15300, 15301, 100000]
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    got = engine.digest32_batch(data, off)
    for i, ln in enumerate(lens):
        assert got[i].tobytes() == hashlib.sha512(data[int(off[i]):int(off[i + 1])].tobytes()).digest()[:32], ln
    for k in golden["digest_kats"]:
        m = bytes.fromhex(k["msg"])
        out = engine.digest32_batch(m, np.array([0, len(m)], dtype=np.uint64))
        assert out[0].tobytes().hex() == k["sha512"][:64]
    # the reference's mempool fixture (mempool/src/tests/common.rs:65-77)
    sb = bytes.fromhex(golden["reference"]["serialized_batch"])
    assert engine.digest32_batch(sb, np.array([0, len(sb)], np.uint64))[0].tobytes().hex() == golden["reference"]["batch_digest"]


def test_full_size_2pow20_properties(engine, oracle):
    """BASELINE config 2 at full size (2^20 records): size-independent properties instead of 2^20 oracle verifies —
    a 4,096-record signed base set is tiled 256x; ~1 % of the records get a seeded bit flip.  Expected bitmap = all
    ones except the corrupted positions, whose verdicts are recomputed by the oracle (about 10 k verifies)."""
    base = make_workload(oracle, 4096, n_keys=4096, seed=77)
    recs = np.tile(to_rec128(base), (256, 1))
    n = recs.shape[0]
    assert n == 1 << 20
    rng = np.random.default_rng(78)
    bad = rng.choice(n, n // 100, replace=False)
    byte = rng.integers(0, 128, bad.shape[0])
    bit = rng.integers(0, 8, bad.shape[0])
    recs[bad, byte] ^= (1 << bit).astype(np.uint8)
    got = engine.verify_rec128(recs)
    want = np.ones(n, dtype=bool)
    want[bad] = oracle.verify_rec128(recs[bad])
    assert (got == want).all()
    assert got.sum() == n - (~want).sum()


def test_registered_committee_lookup_mixed_with_unknown_keys(engine, oracle):
    """With a committee registered, entry points that receive key BYTES resolve them on the device: registered keys take
    the table path, unknown keys the generic path — same verdicts, including adversarial keys that collide in nothing."""
    rng = np.random.default_rng(55)
    w = make_workload(oracle, 3000, n_keys=64, seed=56, corrupt_frac=0.05)
    recs = to_rec128(w)
    engine.committee_register(w["pks"][:40])          # 24 of the 64 signer keys stay unknown
    want = oracle.verify_rec128(recs)
    assert (engine.verify_rec128(recs) == want).all()
    assert (engine.verify_rec128(recs, mode=1) == oracle.verify_rec128(recs, mode=1)).all()
    got = engine.verify_var(w["sig"], w["pk"], w["msgs"], w["off"])
    assert (got == want).all()
    # reference-shaped call with on-GPU Digest, both key forms
    msgs = rng.integers(0, 256, (3000, 200), dtype=np.uint8)
    d = oracle.digest32_batch(msgs.reshape(-1), np.arange(3001, dtype=np.uint64) * 200)
    sig = oracle.sign_batch(w["seeds"], w["pks"], w["key_idx"], d.reshape(-1), np.arange(3001, dtype=np.uint64) * 32)
    sig[::17, 3] ^= 0x40
    want2 = oracle.verify_rec128(np.concatenate([sig, w["pks"][w["key_idx"]], d], axis=1))
    assert (engine.verify_msgs(sig, msgs.reshape(-1), 200, pk=w["pks"][w["key_idx"]]) == want2).all()
    engine.committee_register(w["pks"])
    assert (engine.verify_msgs(sig, msgs.reshape(-1), 200, validator_idx=w["key_idx"]) == want2).all()
    assert (engine.verify_msgs(sig, msgs.reshape(-1), 200, pk=w["pks"][w["key_idx"]]) == want2).all()
    engine.committee_register(np.zeros((0, 32), np.uint8))   # clear the committee again for later tests
    assert (engine.verify_rec128(recs) == want).all()


def test_verify_msgs_chunked_pipeline(engine, oracle):
    """hs_verify_msgs splits large calls into 2^17-record chunks on two streams; verdicts must not depend on the split."""
    n = (1 << 17) * 2 + 777
    base = make_workload(oracle, 2048, n_keys=2048, seed=91, msg_len=96)
    reps = (n + 2047) // 2048
    msgs = np.tile(base["msgs"].reshape(2048, 96), (reps, 1))[:n]
    d = oracle.digest32_batch(base["msgs"], np.arange(2049, dtype=np.uint64) * 96)
    sig_base = oracle.sign_batch(base["seeds"], base["pks"], base["key_idx"], d.reshape(-1), np.arange(2049, dtype=np.uint64) * 32)
    sig = np.tile(sig_base, (reps, 1))[:n].copy()
    pk = np.tile(base["pks"][base["key_idx"]], (reps, 1))[:n].copy()
    rng = np.random.default_rng(92)
    bad = rng.choice(n, 3000, replace=False)
    sig[bad, rng.integers(0, 64, 3000)] ^= 1
    got = engine.verify_msgs(sig, msgs.reshape(-1), 96, pk=pk)
    want = np.ones(n, dtype=bool)
    want[bad] = False
    assert (got == want).all()


@pytest.mark.parametrize("base_window,key_window", [(8, 8), (12, 10), (16, 12), (20, 14), (24, 16), (24, 15), (24, 13), (24, 14), (24, 9), (24, 11), (22, 12), (26, 15), (24, 17), (24, 12)])
def test_window_width_independence(oracle, golden, base_window, key_window):
    """Verdicts must not depend on the comb window widths (table sizes): golden vectors + a random set + the randomised
    adversarial set, through the generic, lookup, indexed and hs_verify_qcs paths — for the small / medium table geometries AND
    the ones the benchmarks run on an 80 GB H100 (base 24 with key windows 13 = 4,096 keys, 12 = 10,000 keys, 14, 15, and 9 / 11, where
    253 mod w hits the recoder's extra-digit cases)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine
    e = Engine(0, base_window=base_window, key_window=key_window)
    try:
        vs, sig, pk, msgs = _golden_arrays(golden, only32=True)
        recs = np.concatenate([sig, pk, np.array([np.frombuffer(m, np.uint8) for m in msgs])], axis=1)
        got = e.verify_rec128(recs)
        for v, a in zip(vs, got):
            assert bool(a) == v["strict"], v["name"]
        w = make_workload(oracle, 2000, n_keys=37, seed=300 + base_window, corrupt_frac=0.05)
        r = to_rec128(w)
        want = oracle.verify_rec128(r)
        assert (e.verify_rec128(r) == want).all()
        assert e.committee_register(w["pks"]).all()
        assert (e.verify_rec128(r) == want).all()                      # lookup path
        keys, inv = np.unique(pk, axis=0, return_inverse=True)
        e.committee_register(keys)
        assert e.window_bits == (key_window, base_window)
        got = e.verify_committee(inv.astype(np.uint32), sig, recs[:, 96:], msg_idx=np.arange(len(vs), dtype=np.uint32))
        for v, a in zip(vs, got):
            assert bool(a) == v["strict"], v["name"]
        got = e.verify_rec128(recs, mode=1)                                 # golden vectors through the lookup path, batch-eq
        for v, a in zip(vs, got):
            assert bool(a) == v["batch_eq"], v["name"]
        # randomised adversarial records: lookup (all keys registered), indexed, and one-call QC verification
        from oracle_api import make_adversarial
        adv = make_adversarial(oracle, 4000, seed=500 + 31 * base_window + key_window)
        ws, we = oracle.verify_rec128(adv, mode=0), oracle.verify_rec128(adv, mode=1)
        akeys, ainv = np.unique(adv[:, 64:96], axis=0, return_inverse=True)
        e.committee_register(akeys)
        assert (e.verify_rec128(adv, mode=0) == ws).all() and (e.verify_rec128(adv, mode=1) == we).all()
        got = e.verify_committee(ainv.astype(np.uint32), adv[:, :64].copy(), adv[:, 96:].copy(), msg_idx=np.arange(len(adv), dtype=np.uint32), mode=0)
        assert (got == ws).all()
        _check_qcs_against_oracle(e, oracle, n_val=23, n_qc=60, seed=key_window)
    finally:
        e.close()


def _check_qcs_against_oracle(e, oracle, n_val, n_qc, seed):
    """hs_verify_qcs on a registered committee (indices and key bytes) against the oracle's per-vote batch-eq verdicts."""
    rng = np.random.default_rng(seed)
    seeds = rng.integers(0, 256, (n_val, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    pre = np.zeros((n_qc, 40), dtype=np.uint8)
    pre[:, :32] = rng.integers(0, 256, (n_qc, 32), dtype=np.uint8)
    pre[:, 32:] = np.arange(n_qc, dtype="<u8").view(np.uint8).reshape(n_qc, 8)
    digests = oracle.digest32_batch(pre.reshape(-1), np.arange(n_qc + 1, dtype=np.uint64) * 40)
    qi = np.repeat(np.arange(n_qc, dtype=np.uint32), rng.integers(1, n_val, n_qc))
    n = len(qi)
    vidx = rng.integers(0, n_val, n).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, vidx, digests[qi].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    bad = rng.choice(n, max(1, n // 40), replace=False)
    sig[bad, rng.integers(0, 64, len(bad))] ^= 0x10
    want_votes = oracle.verify_rec128(np.concatenate([sig, pks[vidx], digests[qi]], axis=1), mode=1)
    want_qc = np.ones(n_qc, dtype=bool)
    np.logical_and.at(want_qc, qi, want_votes)
    e.committee_register(pks)
    got_qc, got_votes = e.verify_qcs(pre, sig, qi, validator_idx=vidx, want_votes=True)
    assert (got_votes == want_votes).all() and (got_qc == want_qc).all()
    assert (e.verify_qcs(pre, sig, qi, pk=pks[vidx]) == want_qc).all()


@pytest.mark.parametrize("n_keys,expect_window", [(4096, 13), (10000, 12)])
def test_benchmark_sized_committees_with_adversarial_members(engine, oracle, n_keys, expect_window):
    """The committee sizes of BASELINE configs [1]/[2] (4,096 keys -> 13-bit key windows, 34 GB of tables on an 80 GB H100) and
    [3] (10,000 keys -> 12-bit, 46 GB): honest keys plus the adversarial generator's keys (mixed order, small order, non-decompressible, non-canonical)
    registered together; honest + corrupted + adversarial records through the lookup and the indexed path, bit-exact against
    the oracle."""
    from hotstuff_b200 import Engine
    from oracle_api import make_adversarial
    engine.committee_register(np.zeros((0, 32), np.uint8))      # release the session engine's tables: this test needs the HBM
    w = make_workload(oracle, 20000, n_keys=n_keys - 600, seed=9000 + n_keys, corrupt_frac=0.03)
    adv = make_adversarial(oracle, 6000, seed=n_keys)
    akeys = np.unique(adv[:, 64:96], axis=0)[:600]
    keys = np.concatenate([w["pks"], akeys], axis=0)
    keys = keys[np.random.default_rng(1).permutation(len(keys))]
    assert len(np.unique(keys, axis=0)) == len(keys) <= n_keys
    recs = np.concatenate([to_rec128(w), adv], axis=0)
    ws, we = oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)
    e = Engine(0)
    try:
        valid = e.committee_register(keys)
        assert e.window_bits == (expect_window, 24)
        assert (valid == np.array([oracle.decompress_ok(k.tobytes()) for k in keys])).all()
        assert (e.verify_rec128(recs, mode=0) == ws).all()           # lookup path; keys outside the 600 take the generic pass
        assert (e.verify_rec128(recs, mode=1) == we).all()
        index_of = {k.tobytes(): i for i, k in enumerate(keys)}
        known = np.array([r[64:96].tobytes() in index_of for r in recs])
        vidx = np.array([index_of.get(r[64:96].tobytes(), 0) for r in recs], dtype=np.uint32)
        got = e.verify_committee(vidx[known], recs[known, :64].copy(), recs[known, 96:].copy(), msg_idx=np.arange(int(known.sum()), dtype=np.uint32))
        assert (got == ws[known]).all() and known.sum() > 20000
        # incremental epoch change: drop 5 validators, add 3 new ones + one that is already there
        seeds = np.random.default_rng(2).integers(0, 256, (3, 32), dtype=np.uint8)
        newpk = oracle.keygen_batch(seeds)
        removed = np.unique(vidx[known][vidx[known] != 7])[:5]
        idx = e.committee_update(add=np.concatenate([newpk, keys[7:8]]), remove=removed)
        assert idx[3] == 7 and set(idx[:3]) <= set(removed) | set(range(len(keys), len(keys) + 3))   # freed or spare slots
        m = np.random.default_rng(3).integers(0, 256, (3, 32), dtype=np.uint8)
        sg = oracle.sign_batch(seeds, newpk, np.arange(3, dtype=np.uint32), m.reshape(-1), np.arange(4, dtype=np.uint64) * 32)
        assert e.verify_committee(idx[:3], sg, m, msg_idx=np.arange(3, dtype=np.uint32)).all()          # new validators verify by index
        assert e.verify_rec128(np.concatenate([sg, newpk, m], axis=1)).all()                            # ... and by key bytes
        got = e.verify_committee(vidx[known], recs[known, :64].copy(), recs[known, 96:].copy(), msg_idx=np.arange(int(known.sum()), dtype=np.uint32))
        gone = np.isin(vidx[known], removed)                                                            # dead slot, or now someone else's key
        assert gone.any() and not got[gone].any() and (got[~gone] == ws[known][~gone]).all()
        assert (e.verify_rec128(recs, mode=0) == ws).all()            # by key bytes a removed key is simply unregistered: generic path
    finally:
        e.close()


def test_concurrent_callers_share_one_context(engine, oracle):
    """SURVEY §8b threading: the Core task and two Processor tasks call into the crate concurrently; a context must serve
    >= 3 concurrent callers.  Four Python threads (ctypes drops the GIL) hammer different entry points of ONE context."""
    import threading
    w = make_workload(oracle, 1500, n_keys=13, seed=404, corrupt_frac=0.1)
    recs = to_rec128(w)
    want = oracle.verify_rec128(recs)
    digest = oracle.digest32(b"shared")
    msgs = np.tile(np.frombuffer(digest, np.uint8), 13)
    sig = oracle.sign_batch(w["seeds"], w["pks"], np.arange(13, dtype=np.uint32), msgs, np.arange(14, dtype=np.uint64) * 32)
    votes = np.concatenate([w["pks"], sig], axis=1)
    blob = np.random.default_rng(1).integers(0, 256, 40000, dtype=np.uint8)
    off = np.array([0, 100, 15400, 40000], dtype=np.uint64)
    want_d = oracle.digest32_batch(blob, off)
    errors = []

    def worker(kind):
        try:
            for _ in range(12):
                if kind == 0:
                    assert (engine.verify_rec128(recs) == want).all()
                elif kind == 1:
                    assert engine.verify_batch_shared_msg(digest, votes) is True
                elif kind == 2:
                    assert (engine.digest32_batch(blob, off) == want_d).all()
                else:
                    assert (engine.verify_var(w["sig"], w["pk"], w["msgs"], w["off"]) == want).all()
        except Exception as ex:  # noqa: BLE001
            errors.append((kind, repr(ex)))

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_verify_msgs_unaligned_message_lengths(engine, oracle):
    """Reference-shaped call with the reference's own transaction size (100 B, mempool/src/tests/common.rs:55-62) and odd lengths."""
    for L in (100, 1, 77, 513):
        n = 300
        rng = np.random.default_rng(L)
        seeds = rng.integers(0, 256, (5, 32), dtype=np.uint8)
        pks = oracle.keygen_batch(seeds)
        kidx = (np.arange(n) % 5).astype(np.uint32)
        msgs = rng.integers(0, 256, (n, L), dtype=np.uint8)
        d = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
        sig = oracle.sign_batch(seeds, pks, kidx, d.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
        sig[::9, 10] ^= 4
        want = oracle.verify_rec128(np.concatenate([sig, pks[kidx], d], axis=1))
        assert (engine.verify_msgs(sig, msgs.reshape(-1), L, pk=pks[kidx]) == want).all(), L


def test_argument_errors_are_reported_not_crashed(engine):
    import ctypes
    lib = engine.lib
    assert lib.hs_verify_rec128(engine.h, None, 5, 0, None) != 0
    assert b"bad argument" in lib.hs_last_error(engine.h)
    assert lib.hs_verify_rec128(engine.h, None, 0, 0, None) == 0          # n == 0 is a no-op
    bm = (ctypes.c_uint32 * 1)()
    rec = (ctypes.c_uint8 * 128)()
    assert lib.hs_verify_rec128(engine.h, rec, 1, 7, bm) != 0            # unknown mode
    import numpy as np
    ok = ctypes.c_int(5)
    assert lib.hs_verify_batch_shared_msg(engine.h, None, None, 0, ctypes.byref(ok), None) != 0   # null digest
    assert ok.value == 5                                                                         # ... and *all_ok is left untouched
    # offsets that go backwards are an argument error, not a device fault
    off = np.array([0, 40, 20, 60], dtype=np.uint64)
    buf = np.zeros(64, np.uint8)
    out = np.zeros((3, 32), np.uint8)
    assert lib.hs_digest32_batch(engine.h, buf.ctypes.data, off.ctypes.data, 3, out.ctypes.data) != 0
    assert b"non-decreasing" in lib.hs_last_error(engine.h)
    # a committee-indexed call without a committee is refused (r1: null-pointer device read)
    engine.committee_register(np.zeros((0, 32), np.uint8))
    vidx = np.zeros(4, np.uint32)
    sig = np.zeros((4, 64), np.uint8)
    bm4 = np.zeros(1, np.uint32)
    assert lib.hs_verify_committee(engine.h, vidx.ctypes.data, sig.ctypes.data, None, buf.ctypes.data, 1, 4, 0, bm4.ctypes.data) != 0


def test_randomised_adversarial_differential(engine, oracle):
    """20 k randomised adversarial records (mixed-order keys and nonces, S + l, small-order points, random encodings, identity
    key, high bits): strict and batch-eq verdicts must equal the oracle's bit for bit, through the generic path, the
    registered-key lookup path and the indexed path."""
    from oracle_api import make_adversarial
    recs = make_adversarial(oracle, 20000, seed=2026)
    want_s = oracle.verify_rec128(recs, mode=0)
    want_e = oracle.verify_rec128(recs, mode=1)
    assert 0.05 < want_s.mean() < 0.6 and (want_e & ~want_s).sum() > 500    # the set really is adversarial
    engine.committee_register(np.zeros((0, 32), np.uint8))
    assert (engine.verify_rec128(recs, mode=0) == want_s).all()
    assert (engine.verify_rec128(recs, mode=1) == want_e).all()
    keys, inv = np.unique(recs[:, 64:96], axis=0, return_inverse=True)
    engine.committee_register(keys[: len(keys) // 2])                       # half of the (mostly weird) keys registered
    assert (engine.verify_rec128(recs, mode=0) == want_s).all()
    assert (engine.verify_rec128(recs, mode=1) == want_e).all()
    engine.committee_register(keys)
    got = engine.verify_committee(inv.astype(np.uint32), recs[:, :64].copy(), recs[:, 96:].copy(), msg_idx=np.arange(len(recs), dtype=np.uint32), mode=0)
    assert (got == want_s).all()
    engine.committee_register(np.zeros((0, 32), np.uint8))


def test_verify_qcs_one_pass(engine, oracle):
    """hs_verify_qcs: QC::digest on the GPU, verify_batch condition per vote, per-QC AND — against the oracle, with key bytes and
    with validator indices, including a certificate without votes and a certificate with one bad vote."""
    rng = np.random.default_rng(808)
    N, Q = 50, 300
    seeds = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    pre = np.zeros((Q, 40), dtype=np.uint8)
    pre[:, :32] = rng.integers(0, 256, (Q, 32), dtype=np.uint8)
    pre[:, 32:] = np.arange(Q, dtype="<u8").view(np.uint8).reshape(Q, 8)
    digests = oracle.digest32_batch(pre.reshape(-1), np.arange(Q + 1, dtype=np.uint64) * 40)
    votes_per = rng.integers(0, 40, Q)
    votes_per[5] = 0
    qi = np.repeat(np.arange(Q, dtype=np.uint32), votes_per)
    n = len(qi)
    vidx = rng.integers(0, N, n).astype(np.uint32)
    sig = oracle.sign_batch(seeds, pks, vidx, digests[qi].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    bad = rng.choice(n, n // 30, replace=False)
    sig[bad, rng.integers(0, 64, len(bad))] ^= 0x08
    want_votes = oracle.verify_rec128(np.concatenate([sig, pks[vidx], digests[qi]], axis=1), mode=1)
    want_qc = np.ones(Q, dtype=bool)
    np.logical_and.at(want_qc, qi, want_votes)
    engine.committee_register(np.zeros((0, 32), np.uint8))
    got_qc, got_votes = engine.verify_qcs(pre, sig, qi, pk=pks[vidx], want_votes=True)
    assert (got_votes == want_votes).all() and (got_qc == want_qc).all() and got_qc[5] and (~want_qc).sum() > 20
    engine.committee_register(pks)
    assert (engine.verify_qcs(pre, sig, qi, validator_idx=vidx) == want_qc).all()
    assert (engine.verify_qcs(pre, sig, qi, pk=pks[vidx]) == want_qc).all()
    engine.committee_register(np.zeros((0, 32), np.uint8))


def test_key_cache_learns_unregistered_keys(oracle):
    """Nothing registered: the first sighting of a key takes the generic path, the engine builds its table between calls, and
    later calls take the table path — verdicts identical throughout (honest, corrupted and adversarial keys alike)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine
    from oracle_api import make_adversarial
    e = Engine(0, base_window=12)
    try:
        w = make_workload(oracle, 6000, n_keys=40, seed=606, corrupt_frac=0.05)
        recs = to_rec128(w)
        want = oracle.verify_rec128(recs)
        assert e.cached_keys == 0
        for rep in range(4):
            assert (e.verify_rec128(recs) == want).all(), rep
        assert e.cached_keys >= 40
        got = e.verify_var(w["sig"], w["pk"], w["msgs"], w["off"])
        assert (got == want).all()
        adv = make_adversarial(oracle, 3000, seed=99)
        ws, we = oracle.verify_rec128(adv, mode=0), oracle.verify_rec128(adv, mode=1)
        for rep in range(3):                                   # adversarial keys get cached too; flags must carry over
            assert (e.verify_rec128(adv, mode=0) == ws).all(), rep
            assert (e.verify_rec128(adv, mode=1) == we).all(), rep
        n_cached = e.cached_keys
        assert n_cached > 40
        # an explicit committee switches learning off; clearing it switches learning back on with an empty cache
        e.committee_register(w["pks"])
        assert e.cached_keys == 0 and (e.verify_rec128(recs) == want).all()
        e.committee_register(np.zeros((0, 32), np.uint8))
        for rep in range(3):
            assert (e.verify_rec128(recs) == want).all()
        assert e.cached_keys >= 40
    finally:
        e.close()
    e2 = Engine(0, base_window=12, key_cache=False)
    try:
        for rep in range(3):
            assert (e2.verify_rec128(recs) == want).all()
        assert e2.cached_keys == 0
    finally:
        e2.close()


def test_key_cache_resets_when_the_key_set_rotates(oracle, monkeypatch):
    """A full cache that misses on most of a pass (validator-set rotation) is cleared and relearns."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine
    e = Engine(0, base_window=12, key_window=8)
    try:
        cap = 4096
        a = make_workload(oracle, 2 * cap, n_keys=cap, seed=1)          # exactly fills the cache
        ra, wa_ = to_rec128(a), None
        wa_ = oracle.verify_rec128(ra)
        for _ in range(8):                                                # at most 1,024 new tables are built per call
            assert (e.verify_rec128(ra) == wa_).all()
            if e.cached_keys == cap:
                break
        assert e.cached_keys == cap
        b = make_workload(oracle, 3000, n_keys=50, seed=2)               # a different key set
        rb = to_rec128(b)
        wb = oracle.verify_rec128(rb)
        for _ in range(5):
            assert (e.verify_rec128(rb) == wb).all()
        assert 50 <= e.cached_keys < cap                                 # reset happened, the new set was learned
    finally:
        e.close()


def test_latency_path_small_batches(engine, oracle, golden):
    """n <= 64 with every key registered takes the one-launch latency path (k_verify_small: one warp sums the table entries with
    a shuffle tree, a second warp decompresses R, projective compare).  Golden vectors (incl. the speccheck classes), random
    and adversarial records in calls of 1 .. 64 records through hs_verify_rec128 / hs_verify_committee /
    hs_verify_batch_shared_msg must give the oracle's verdicts, and the same verdicts as the throughput path (n > 64)."""
    from oracle_api import make_adversarial
    vs, sig, pk, msgs = _golden_arrays(golden, only32=True)
    recs = np.concatenate([sig, pk, np.array([np.frombuffer(m, np.uint8) for m in msgs])], axis=1)
    adv = make_adversarial(oracle, 1500, seed=4242)
    w = make_workload(oracle, 500, n_keys=9, seed=4243, corrupt_frac=0.2)
    allrecs = np.concatenate([recs, adv, to_rec128(w)], axis=0)
    ws, we = oracle.verify_rec128(allrecs, mode=0), oracle.verify_rec128(allrecs, mode=1)
    keys, inv = np.unique(allrecs[:, 64:96], axis=0, return_inverse=True)
    engine.committee_register(keys)
    l0 = engine.kernel_launches
    assert (engine.verify_rec128(allrecs[:64], mode=0) == ws[:64]).all()
    assert engine.kernel_launches - l0 == 1, "n = 64 with registered keys must be ONE kernel launch"
    assert (engine.verify_rec128(allrecs, mode=0) == ws).all()            # throughput path, same inputs
    sizes = [1, 2, 3, 5, 31, 32, 33, 64]
    lo, k = 0, 0
    while lo < len(allrecs):
        n = sizes[k % len(sizes)]
        k += 1
        chunk = allrecs[lo:lo + n]
        assert (engine.verify_rec128(chunk, mode=0) == ws[lo:lo + n]).all(), lo
        assert (engine.verify_rec128(chunk, mode=1) == we[lo:lo + n]).all(), lo
        got = engine.verify_committee(inv[lo:lo + n].astype(np.uint32), chunk[:, :64].copy(), chunk[:, 96:].copy(), msg_idx=np.arange(len(chunk), dtype=np.uint32), mode=0)
        assert (got == ws[lo:lo + n]).all(), lo
        lo += n
    # unknown authority index on the latency path -> reject
    assert not engine.verify_committee(np.array([len(keys) + 9], dtype=np.uint32), allrecs[:1, :64].copy(), allrecs[:1, 96:].copy())[0]
    # QC of a 4-node committee (3 votes over one digest), valid and with one bad vote
    seeds = np.random.default_rng(5).integers(0, 256, (4, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    engine.committee_register(pks)
    d = oracle.digest32(bytes(32) + (3).to_bytes(8, "little"))
    sg = oracle.sign_batch(seeds, pks, np.arange(4, dtype=np.uint32), np.tile(np.frombuffer(d, np.uint8), 4), np.arange(5, dtype=np.uint64) * 32)
    votes = np.concatenate([pks[1:], sg[1:]], axis=1)
    l0 = engine.kernel_launches
    assert engine.verify_batch_shared_msg(d, votes) is True and engine.kernel_launches - l0 == 1
    votes[1, 40] ^= 1
    ok, bits = engine.verify_batch_shared_msg(d, votes, want_bitmap=True)
    assert ok is False and list(bits) == [True, False, True]
    # a key that is not registered falls back to the throughput path, same verdict
    other = make_workload(oracle, 3, n_keys=3, seed=77)
    assert engine.verify_rec128(to_rec128(other)).all()
    engine.committee_register(np.zeros((0, 32), np.uint8))


def test_long_message_digest_kernel(engine):
    """hs_digest32_batch with a few long messages (mempool batches, ~15 kB) runs the warp-cooperative kernel."""
    rng = np.random.default_rng(15)
    lens = [15300, 15301, 1024, 4096, 128 * 33, 128 * 64 + 5, 100000, 2000]
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    got = engine.digest32_batch(data, off)
    for i, ln in enumerate(lens):
        assert got[i].tobytes() == hashlib.sha512(data[int(off[i]):int(off[i + 1])].tobytes()).digest()[:32], ln
    one = engine.digest32_batch(data[:15300], np.array([0, 15300], dtype=np.uint64))
    assert one[0].tobytes() == hashlib.sha512(data[:15300].tobytes()).digest()[:32]


def test_fixed_length_digest_kernel_shapes(engine, oracle):
    """hs_verify_msgs with 16-byte aligned message sizes takes the staged digest kernel (k_digest32_fixed): multiples of 128
    (constant padding block) and others (generic tail), ragged record counts."""
    for L, n in ((512, 1000), (128, 33), (256, 4097), (144, 500), (640, 31), (1040, 200)):
        rng = np.random.default_rng(L)
        seeds = rng.integers(0, 256, (7, 32), dtype=np.uint8)
        pks = oracle.keygen_batch(seeds)
        kidx = (np.arange(n) % 7).astype(np.uint32)
        msgs = rng.integers(0, 256, (n, L), dtype=np.uint8)
        d = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
        sig = oracle.sign_batch(seeds, pks, kidx, d.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
        sig[::11, 20] ^= 2
        want = oracle.verify_rec128(np.concatenate([sig, pks[kidx], d], axis=1))
        assert (engine.verify_msgs(sig, msgs.reshape(-1), L, pk=pks[kidx]) == want).all(), (L, n)


def test_gpu_signer_is_byte_identical_to_rfc8032(engine, oracle, golden):
    """hs_keygen_batch / hs_sign_digests (load generation): deterministic RFC 8032 output, byte for byte the oracle's (which is
    pinned on the RFC 8032 KATs and OpenSSL), including the reference's keys() and its "Hello, world!" signature."""
    r = golden["reference"]
    seeds = np.array([np.frombuffer(bytes.fromhex(s), np.uint8) for s in r["seeds"]])
    pks = engine.keygen_batch(seeds)
    assert [p.tobytes().hex() for p in pks] == r["pks"]
    hello = np.frombuffer(bytes.fromhex(r["hello_digest"]), np.uint8).reshape(1, 32)
    assert engine.sign_digests(seeds, pks, hello, key_idx=[3])[0].tobytes().hex() == r["hello_sig_key3"]
    rng = np.random.default_rng(99)
    n, nk = 5000, 300
    sd = rng.integers(0, 256, (nk, 32), dtype=np.uint8)
    pk = engine.keygen_batch(sd)
    assert (pk == oracle.keygen_batch(sd)).all()
    ki = rng.integers(0, nk, n).astype(np.uint32)
    dg = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sig = engine.sign_digests(sd, pk, dg, key_idx=ki)
    assert (sig == oracle.sign_batch(sd, pk, ki, dg.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)).all()
    assert engine.verify_rec128(np.concatenate([sig, pk[ki], dg], axis=1)).all()


def test_deferred_results_mode(oracle):
    """hs_set_deferred: the finish kernel of pass i runs on the engine's tail stream beside the main kernel of pass i+1 (two scratch
    sets alternate).  Twelve back-to-back passes with different inputs and sizes, no synchronisation in between; every pass's bitmap
    and per-QC AND must equal the oracle after hs_results_wait()."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine
    e = Engine(0, base_window=16)
    try:
        dev = torch.device("cuda", 0)
        rng = np.random.default_rng(77)
        N, Q = 60, 40
        seeds = rng.integers(0, 256, (N, 32), dtype=np.uint8)
        pks = oracle.keygen_batch(seeds)
        assert e.committee_register(pks).all()
        passes = []
        for p in range(12):
            n = int(rng.integers(500, 9000))
            pre = rng.integers(0, 256, (Q, 40), dtype=np.uint8)
            dig = oracle.digest32_batch(pre.reshape(-1), np.arange(Q + 1, dtype=np.uint64) * 40)
            qi = rng.integers(0, Q, n).astype(np.uint32)
            vi = rng.integers(0, N, n).astype(np.uint32)
            sig = oracle.sign_batch(seeds, pks, vi, dig[qi].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
            bad = rng.choice(n, n // 20, replace=False)
            sig[bad, rng.integers(0, 64, len(bad))] ^= 0x20
            want = oracle.verify_rec128(np.concatenate([sig, pks[vi], dig[qi]], axis=1), mode=1)
            want_qc = np.ones(Q, dtype=bool)
            np.logical_and.at(want_qc, qi, want)
            t = dict(n=n, want=want, want_qc=want_qc, d_pre=torch.from_numpy(pre.reshape(-1)).to(dev), d_dig=torch.empty((Q, 32), dtype=torch.uint8, device=dev),
                     d_sig=torch.from_numpy(sig).to(dev), d_vi=torch.from_numpy(vi.astype(np.int32)).to(dev), d_qi=torch.from_numpy(qi.astype(np.int32)).to(dev),
                     d_bm=torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev), d_qc=torch.zeros((Q + 31) // 32, dtype=torch.int32, device=dev))
            passes.append(t)
        e.set_deferred(True)
        for t in passes:
            e.digest32_fixed_dev(t["d_pre"], 40, t["d_dig"], Q)
            e.verify_qc_votes_dev(t["d_dig"], t["d_sig"], t["d_qi"], t["d_bm"], t["n"], d_vidx=t["d_vi"])
            e.qc_and_dev(t["d_bm"], t["d_qi"], t["n"], Q, t["d_qc"])
        e.results_wait()
        torch.cuda.synchronize()
        e.set_deferred(False)
        for k, t in enumerate(passes):
            bits = np.unpackbits(t["d_bm"].cpu().numpy().view(np.uint8), bitorder="little")[:t["n"]].astype(bool)
            qcb = np.unpackbits(t["d_qc"].cpu().numpy().view(np.uint8), bitorder="little")[:Q].astype(bool)
            assert (bits == t["want"]).all() and (qcb == t["want_qc"]).all(), k
    finally:
        e.close()
