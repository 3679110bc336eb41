"""Every device-resident entry point, enqueued on a stream the caller created, bit for bit against the CPU oracle and hashlib.

The `_dev` calls are the throughput interface: they take device pointers and a cudaStream_t and return once their work is enqueued.
Three things are checked here that the host-pointer calls, which always run on the context's own stream, cannot show:

- Stream order.  The inputs of each call are garbage (zero signatures, zero seeds, shifted message bytes) until the caller's stream
  copies the true ones in behind a ~0.2 s sleep kernel.  Any engine work not ordered after the caller's earlier work on that stream
  reads the garbage and the verdicts differ, whatever the timing.
- Parity at the shapes where the paths differ: 1, 31, 32, 33 and 4,097 records and one pass past 2^18 (finish group of 8); message
  lengths on both sides of each SHA-512 padding boundary of R || A || M, and of each Digest kernel; removed committee slots and indices
  past the committee; 5 % of keys outside the committee, which take the side stream and join back before the finish kernel; n == 0.
- Scratch ownership between a `_dev` pass and the host-pointer calls that follow it on the same thread: the host call waits for the
  pass that still reads the shared verify scratch, and the latency path (own scratch) does not.

Every bitmap starts filled with a sentinel, one guard word past its end; every call is checked on all n bits, on the unused high bits
of its last word (0) and on the guard word (untouched)."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle_api import L_ORDER, make_adversarial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, FOREIGN = 256, 16                       # committee keys, then keys that are never registered
REMOVED = np.array([3, 77, 200], np.uint32)  # committee slots removed by committee_update in the committee fixture
SPARES = 16                                # spare slots a registration reserves (at least 16): indices K .. K + 15 hold no key
SIZES = [1, 31, 32, 33, 4097]
FIN8_N = (1 << 18) + 5                     # run_verify: 2^18 <= n < 2^19 records -> 8 records per finish thread
VAR_LENS = [0, 1, 47, 48, 63, 64, 111, 112, 175, 176, 300]  # 64 + len: 111 | 112 and 239 | 240 bytes of R || A || M
MSG_LENS = [1, 32, 40, 112, 128, 240, 512]  # generic Digest reader (< 128 or not a multiple of 16), staged with tail, staged constant pad
SLEEP = 400_000_000                        # cycles: about 0.2 s at H100 clocks
LONG_SLEEP = 1_000_000_000                 # about 0.5 s
BIG = 1 << 20
SENTINEL = 0xA5A5A5A5
TABLE_BUDGET = 4 << 30                     # per-key tables of each fresh context (the session context may hold its own)

IDENTITY = (1).to_bytes(32, "little")
B_ENC = int("6666666666666666666666666666666666666666666666666666666666666658", 16).to_bytes(32, "little")


# ---------------------------------------------------------------------------------------------------- signed sets (CPU)
def _secret(seed):
    h = hashlib.sha512(bytes(seed)).digest()
    return int.from_bytes(bytes([h[0] & 248]) + h[1:31] + bytes([(h[31] & 127) | 64]), "little"), h[32:]


def _sha_k(oracle, r_enc, a_enc, m):
    return oracle.sc_reduce64(hashlib.sha512(bytes(r_enc) + bytes(a_enc) + bytes(m)).digest())


def sign_msgs(oracle, keys, kidx, msgs, off, rng, corrupt=0.03, eq_only=0.03):
    """Signatures of message i (msgs[off[i]:off[i+1]]) by key kidx[i]; `eq_only` of them become R = the identity, S = k * a (the
    cofactorless equation holds: batch-eq accepts, strict rejects) and `corrupt` of the rest get one flipped signature bit."""
    seeds, pks = keys
    n = len(kidx)
    sig = oracle.sign_batch(seeds, pks, kidx, msgs, off)
    pick = rng.permutation(n)
    n_eq, n_bad = int(n * eq_only), int(n * corrupt)
    for i in pick[:n_eq]:
        a, _ = _secret(seeds[kidx[i]])
        k = _sha_k(oracle, IDENTITY, pks[kidx[i]], msgs[int(off[i]):int(off[i + 1])])
        sig[i] = np.frombuffer(IDENTITY + (k * a % L_ORDER).to_bytes(32, "little"), np.uint8)
    for i in pick[n_eq:n_eq + n_bad]:
        sig[i, int(rng.integers(64))] ^= np.uint8(1 << int(rng.integers(8)))
    return sig


def sign_digests(oracle, keys, kidx, digests, rng, **kw):
    n = len(kidx)
    return sign_msgs(oracle, keys, kidx, np.ascontiguousarray(digests).reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32, rng, **kw)


_REC_CACHE = {}


def rec_set(oracle, keys, n, seed, key_lo=0, key_hi=K, adversarial=True):
    """n rec128 records over 32-byte messages by keys [key_lo, key_hi), with the classes of sign_msgs and, when `adversarial`, an eighth
    of them (capped at 256) replaced by make_adversarial's records at seeded positions."""
    ck = (n, seed, key_lo, key_hi, adversarial)
    if ck not in _REC_CACHE:
        rng = np.random.default_rng(seed)
        kidx = rng.integers(key_lo, key_hi, n).astype(np.uint32)
        msgs = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        sig = sign_digests(oracle, keys, kidx, msgs, rng)
        recs = np.concatenate([sig, keys[1][kidx], msgs], axis=1)
        n_adv = min(n // 8, 256) if adversarial else 0
        if n_adv:
            recs[rng.choice(n, n_adv, replace=False)] = make_adversarial(oracle, n_adv, seed=seed)
        _REC_CACHE[ck] = recs
    return _REC_CACHE[ck]


def tiled(oracle, keys, n, seed, mode=0, **kw):
    """n records tiled from a base set of 4,099 (not a multiple of 32, so no word repeats) and their oracle verdicts."""
    base = rec_set(oracle, keys, 4099, seed, **kw)
    return np.resize(base, (n, 128)), np.resize(oracle.verify_rec128(base, mode), n)


def digest(m):
    return np.frombuffer(hashlib.sha512(bytes(m)).digest()[:32], np.uint8)


# ---------------------------------------------------------------------------------------------------- device helpers
def _torch():
    import torch
    return torch


def dev(a):
    """A device copy of numpy array a (uint32 / uint64 as int32 / int64), on torch's current stream."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint32:
        a = a.view(np.int32)
    elif a.dtype == np.uint64:
        a = a.view(np.int64)
    return _torch().from_numpy(a.copy()).cuda()


def garbage(src, shift=False):
    """Wrong contents of src's shape: zeros, or src's bytes shifted by one."""
    torch = _torch()
    return torch.roll(src, 1) if shift else torch.zeros_like(src)


def land(pairs, cycles=SLEEP):
    """On torch's current stream: a sleep kernel, then the true contents copied over each garbage buffer."""
    _torch().cuda._sleep(cycles)
    for dst, src in pairs:
        dst.copy_(src)


def bitmap(n):
    """(n + 31) / 32 words and one guard word, all SENTINEL, on torch's current stream."""
    torch = _torch()
    return torch.full(((n + 31) // 32 + 1,), int(np.array([SENTINEL], np.uint32).view(np.int32)[0]), dtype=torch.int32, device="cuda")


def words(bools):
    n = len(bools)
    b = np.zeros(((n + 31) // 32) * 32, np.uint8)
    b[:n] = np.asarray(bools, bool)
    return np.packbits(b, bitorder="little").view(np.uint32)


def check_bitmap(t, want, what):
    got = t.cpu().numpy().view(np.uint32)
    w = (len(want) + 31) // 32
    assert got[w] == SENTINEL, "%s: wrote past its bitmap (guard word %08x)" % (what, got[w])
    exp = words(want)
    if not np.array_equal(got[:w], exp):
        bits = np.unpackbits(got[:w].view(np.uint8), bitorder="little")
        bad = np.flatnonzero(bits[:len(want)] != np.asarray(want, bool))
        hi = [j for j in range(w) if got[j] != exp[j]]
        raise AssertionError("%s: %d of %d verdicts differ from the oracle (first at %s); words differing: %s" % (
            what, bad.size, len(want), bad[:8].tolist(), hi[:8]))


def untouched(t, what):
    got = t.cpu().numpy().view(np.uint32)
    assert (got == SENTINEL).all(), "%s: an empty call wrote to its output" % what


def fresh_engine(keys=None, remove=None):
    from hotstuff_b200 import Engine
    e = Engine(0)
    e.set_table_budget(TABLE_BUDGET)
    if keys is not None:
        assert e.committee_register(keys[1][:K]).all()
        if remove is not None:
            e.committee_update(remove=remove)
    return e


def live_mask():
    live = np.zeros(K + SPARES + 1, bool)
    live[:K] = True
    live[REMOVED] = False
    return live


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(9090)
    seeds = rng.integers(0, 256, size=(K + FOREIGN, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


@pytest.fixture
def s():
    """A non-default stream, made torch's current stream for the test."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        yield st
    st.synchronize()


@pytest.fixture(scope="module")
def committee(keys):
    """A fresh context with the K keys registered in order (committee index = key index) and the REMOVED slots taken out."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import build
    build.build_engine()
    e = fresh_engine(keys, remove=REMOVED)
    yield e
    e.close()


# ---------------------------------------------------------------------------------------------------- CPU
def test_every_device_test_is_marked_gpu():
    import inspect
    mod = sys.modules[__name__]
    for name, fn in inspect.getmembers(mod, inspect.isfunction):
        if not name.startswith("test_"):
            continue
        params = set(inspect.signature(fn).parameters)
        marks = {m.name for m in getattr(fn, "pytestmark", [])}
        if params & {"s", "engine", "committee"}:
            assert "gpu" in marks, "%s uses the device but is not marked gpu" % name


def test_module_skips_cleanly_without_a_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else r.stderr
    assert r.returncode == 0, "without a device the GPU tests did not all skip:\n%s\n%s" % (r.stdout[-3000:], r.stderr[-2000:])
    assert "skipped" in tail and "passed" not in tail and "failed" not in tail and "error" not in tail, tail


def test_group_generator_shares_this_files_keys():
    import test_groups_dev
    assert test_groups_dev.K == K, "test_groups_dev's committee is %d keys, this file registers %d" % (test_groups_dev.K, K)
    assert test_groups_dev.FOREIGN <= FOREIGN, "test_groups_dev signs with %d foreign keys, this file has %d" % (test_groups_dev.FOREIGN, FOREIGN)


def var_set(oracle, keys, rng, lens, reps=3):
    """Records over messages of the given lengths, several per length, in a shuffled order: honest, eq-only (R = identity, S = k * a),
    a flipped signature bit and, for non-empty messages, a flipped message bit after signing.  Returns (sig, pk, msgs, off)."""
    L = np.array([ln for ln in lens for _ in range(4 * reps)])
    L = L[rng.permutation(L.size)]
    n = L.size
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(L)
    msgs = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    sig = sign_msgs(oracle, keys, kidx, msgs, off, rng, corrupt=0.15, eq_only=0.2)
    flip = [i for i in rng.permutation(n)[:n // 6] if L[i] > 0]
    for i in flip:
        msgs[int(off[i]) + int(rng.integers(L[i]))] ^= np.uint8(1 << int(rng.integers(8)))
    return sig, keys[1][kidx].copy(), msgs, off


def test_oracle_at_the_padding_edges_matches_hashlib(oracle, keys):
    """The expectations of the verify_var_dev test: at every padding-edge length, a signature computed here from hashlib's SHA-512
    equals the oracle's, the oracle accepts it in both modes, and rejects it after any single flipped message bit; a signature with
    R = the identity and S = k * a (k from hashlib over R || A || M) is accepted in batch-eq mode only."""
    seeds, pks = keys
    rng = np.random.default_rng(71)
    for ln in VAR_LENS:
        k = int(rng.integers(K))
        a, prefix = _secret(seeds[k])
        A = pks[k].tobytes()
        m = rng.bytes(ln)
        r = int.from_bytes(hashlib.sha512(prefix + m).digest(), "little") % L_ORDER
        R = oracle.scalarmult(r, B_ENC)
        S = (r + _sha_k(oracle, R, A, m) * a) % L_ORDER
        sig = R + S.to_bytes(32, "little")
        assert sig == oracle.sign(seeds[k].tobytes(), m), "length %d: hashlib and the oracle sign differently" % ln
        eq_sig = IDENTITY + (_sha_k(oracle, IDENTITY, A, m) * a % L_ORDER).to_bytes(32, "little")
        cases = [(sig, m, True, True), (eq_sig, m, False, True)]
        if ln:
            bad = bytearray(m)
            bad[int(rng.integers(ln))] ^= 1 << int(rng.integers(8))
            cases.append((sig, bytes(bad), False, False))
        for sg, msg, strict, eq in cases:
            off = np.array([0, len(msg)], np.uint64)
            buf = np.frombuffer(msg, np.uint8)
            got = [bool(oracle.verify_var(np.frombuffer(sg, np.uint8), pks[k], buf, off, mode=md)[0]) for md in (0, 1)]
            assert got == [strict, eq], "length %d: oracle verdicts %s, want %s" % (ln, got, [strict, eq])


# ---------------------------------------------------------------------------------------------------- stream order and parity
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n", SIZES)
def test_rec128_dev(s, engine, oracle, keys, n, mode):
    recs = rec_set(oracle, keys, n, seed=100 + n)
    src = dev(recs)
    d = garbage(src)
    bm = bitmap(n)
    land([(d, src)])
    engine.verify_rec128_dev(d, bm, n, mode)
    s.synchronize()
    check_bitmap(bm, oracle.verify_rec128(recs, mode), "verify_rec128_dev n=%d mode=%d" % (n, mode))


@pytest.mark.gpu
def test_rec128_dev_finish_group_8(s, engine, oracle, keys):
    recs, want = tiled(oracle, keys, FIN8_N, seed=7)
    src = dev(recs)
    d = garbage(src)
    bm = bitmap(FIN8_N)
    land([(d, src)])
    engine.verify_rec128_dev(d, bm, FIN8_N, 0)
    s.synchronize()
    check_bitmap(bm, want, "verify_rec128_dev n=%d" % FIN8_N)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_var_dev_padding_edges(s, engine, oracle, keys, mode):
    sig, pk, msgs, off = var_set(oracle, keys, np.random.default_rng(500 + mode), VAR_LENS)
    n = sig.shape[0]
    want = oracle.verify_var(sig, pk, msgs, off, mode=mode)
    assert want.any() and not want.all()
    skew = 3  # the messages start at odd addresses inside one buffer; sig / pk keep the stager's 16-byte alignment
    buf = np.zeros(skew + msgs.size + 8, np.uint8)
    buf[skew:skew + msgs.size] = msgs
    src_sig, src_pk, src_buf, d_off = dev(sig), dev(pk), dev(buf), dev(off)
    d_sig, d_buf = garbage(src_sig), garbage(src_buf, shift=True)
    bm = bitmap(n)
    land([(d_sig, src_sig), (d_buf, src_buf)])
    engine.verify_var_dev(d_sig, src_pk, d_buf[skew:], d_off, bm, n, mode)
    s.synchronize()
    check_bitmap(bm, want, "verify_var_dev mode=%d" % mode)


def committee_set(oracle, keys, n, rng, n_msgs):
    """Committee votes: validator indices mostly live, some removed slots and some past the committee (spare slots); each vote signed
    by key vidx (any key for an index past the committee) over digests[midx]."""
    vidx = rng.integers(0, K, n).astype(np.uint32)
    if n >= 8:
        pos = rng.choice(n, max(2, n // 16), replace=False)
        half = pos.size // 2
        vidx[pos[:half]] = REMOVED[rng.integers(0, REMOVED.size, half)]
        vidx[pos[half:]] = K + rng.integers(0, SPARES, pos.size - half)
    digests = rng.integers(0, 256, (n_msgs, 32), dtype=np.uint8)
    midx = rng.integers(0, n_msgs, n).astype(np.uint32)
    sig = sign_digests(oracle, keys, vidx % K, digests[midx], rng)
    recs = np.concatenate([sig, keys[1][vidx % K], digests[midx]], axis=1)
    live = live_mask()[vidx]
    return vidx, midx, digests, sig, (oracle.verify_rec128(recs, 0) & live), (oracle.verify_rec128(recs, 1) & live)


@pytest.mark.gpu
@pytest.mark.parametrize("with_midx", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_committee_dev(s, committee, oracle, keys, n, with_midx):
    mode = 1 if with_midx else 0
    vidx, midx, digests, sig, strict, eq = committee_set(oracle, keys, n, np.random.default_rng(200 + n), 7 if with_midx else 1)
    src_sig, src_dig, d_vidx = dev(sig), dev(digests), dev(vidx)
    d_midx = dev(midx) if with_midx else None
    d_sig, d_dig = garbage(src_sig), garbage(src_dig, shift=True)
    bm = bitmap(n)
    land([(d_sig, src_sig), (d_dig, src_dig)])
    committee.verify_committee_dev(d_vidx, d_sig, d_dig, bm, n, d_midx=d_midx, mode=mode)
    s.synchronize()
    check_bitmap(bm, eq if mode else strict, "verify_committee_dev n=%d midx=%s" % (n, with_midx))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [33, 4097])
def test_rec128_dev_lookup_misses_on_the_side_stream(s, committee, oracle, keys, n):
    """Key bytes looked up in the committee on the caller's stream: 5 % of the keys are outside it and take the generic side pass on
    the context's side stream, which must join back into the caller's stream before the finish kernel."""
    rng = np.random.default_rng(300 + n)
    recs = rec_set(oracle, keys, n, seed=300 + n, adversarial=False).copy()
    out = rng.choice(n, max(1, n // 20), replace=False)
    recs[out] = rec_set(oracle, keys, out.size, seed=301 + n, key_lo=K, key_hi=K + FOREIGN, adversarial=False)
    want = oracle.verify_rec128(recs, 0)
    assert want[out].any()
    src = dev(recs)
    d = garbage(src)
    bm = bitmap(n)
    land([(d, src)])
    committee.verify_rec128_dev(d, bm, n, 0)
    s.synchronize()
    check_bitmap(bm, want, "verify_rec128_dev committee lookup n=%d" % n)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pk", "vidx"])
@pytest.mark.parametrize("msg_len", MSG_LENS)
def test_msgs_dev(s, committee, oracle, keys, msg_len, form):
    rng = np.random.default_rng(400 + msg_len)
    n = 97
    msgs = rng.integers(0, 256, (n, msg_len), dtype=np.uint8)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    if form == "vidx":
        kidx[:2] = REMOVED[:2]
    sig = sign_digests(oracle, keys, kidx, np.array([digest(m) for m in msgs]), rng)
    for i in rng.choice(n, 4, replace=False):  # messages changed after signing
        msgs[i, int(rng.integers(msg_len))] ^= np.uint8(1 << int(rng.integers(8)))
    dg = np.array([digest(m) for m in msgs])
    want = oracle.verify_rec128(np.concatenate([sig, keys[1][kidx], dg], axis=1), 0)
    if form == "vidx":
        want &= live_mask()[kidx]
    src_sig, src_msgs = dev(sig), dev(msgs)
    d_sig, d_msgs = garbage(src_sig), garbage(src_msgs, shift=True)
    d_key = dev(keys[1][kidx]) if form == "pk" else dev(kidx)
    d_dig = _torch().full((n, 32), 0xA5, dtype=_torch().uint8, device="cuda")
    bm = bitmap(n)
    land([(d_sig, src_sig), (d_msgs, src_msgs)])
    committee.verify_msgs_dev(d_sig, d_msgs, msg_len, d_dig, bm, n, **({"d_pk": d_key} if form == "pk" else {"d_vidx": d_key}))
    s.synchronize()
    assert np.array_equal(d_dig.cpu().numpy(), dg), "verify_msgs_dev: d_digests != SHA-512(msg)[:32] at msg_len %d" % msg_len
    check_bitmap(bm, want, "verify_msgs_dev msg_len=%d %s" % (msg_len, form))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097])
def test_digest_dev(s, engine, n):
    torch = _torch()
    rng = np.random.default_rng(600 + n)
    lens = rng.integers(0, 301, n)
    lens[:min(n, len(VAR_LENS))] = VAR_LENS[:min(n, len(VAR_LENS))]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]) + 1, dtype=np.uint8)
    want = np.array([digest(data[int(off[i]):int(off[i + 1])]) for i in range(n)])
    src, d_off = dev(data), dev(off)
    d = garbage(src, shift=True)
    out = torch.full((n, 32), 0xA5, dtype=torch.uint8, device="cuda")
    fixed = {ln: rng.integers(0, 256, (n, ln), dtype=np.uint8) for ln in (40, 128)}
    src_fixed = {ln: dev(m) for ln, m in fixed.items()}
    d_fixed = {ln: garbage(t, shift=True) for ln, t in src_fixed.items()}
    out_fixed = {ln: torch.full((n, 32), 0xA5, dtype=torch.uint8, device="cuda") for ln in fixed}
    land([(d, src)] + [(d_fixed[ln], src_fixed[ln]) for ln in fixed])
    engine.digest32_dev(d, d_off, out, n)
    for ln in fixed:
        engine.digest32_fixed_dev(d_fixed[ln], ln, out_fixed[ln], n)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), want), "digest32_dev differs from hashlib"
    for ln, m in fixed.items():
        assert np.array_equal(out_fixed[ln].cpu().numpy(), np.array([digest(r) for r in m])), "digest32_fixed_dev(%d) differs" % ln


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["pk", "vidx"])
def test_qc_votes_dev_and_qc_and_dev(s, committee, oracle, keys, form):
    rng = np.random.default_rng(700 + (form == "vidx"))
    n_qc, n = 9, 1000
    pre = rng.integers(0, 256, (n_qc, 40), dtype=np.uint8)
    qd = np.array([digest(p) for p in pre])
    qi = rng.integers(0, n_qc, n).astype(np.uint32)
    kidx = rng.integers(0, K, n).astype(np.uint32)
    kidx[np.isin(kidx, REMOVED)] = 0  # no removed slot here: each QC is judged by its signatures alone
    sig = sign_digests(oracle, keys, kidx, qd[qi], rng, corrupt=0.0, eq_only=0.02)
    for q in (1, 4):  # two certificates with one bad vote each
        sig[np.flatnonzero(qi == q)[0], 5] ^= 1
    votes = oracle.verify_rec128(np.concatenate([sig, keys[1][kidx], qd[qi]], axis=1), 1)
    qcs = np.ones(n_qc, bool)
    np.logical_and.at(qcs, qi, votes)
    assert qcs.any() and not qcs.all()
    src_sig, src_qd, d_qi = dev(sig), dev(qd), dev(qi)
    d_sig, d_qd = garbage(src_sig), garbage(src_qd, shift=True)
    d_key = dev(keys[1][kidx]) if form == "pk" else dev(kidx)
    vb, qb = bitmap(n), bitmap(n_qc)
    land([(d_sig, src_sig), (d_qd, src_qd)])
    committee.verify_qc_votes_dev(d_qd, d_sig, d_qi, vb, n, **({"d_pk": d_key} if form == "pk" else {"d_vidx": d_key}))
    committee.qc_and_dev(vb, d_qi, n, n_qc, qb)
    s.synchronize()
    check_bitmap(vb, votes, "verify_qc_votes_dev %s" % form)
    check_bitmap(qb, qcs, "qc_and_dev %s" % form)


def group_set(oracle, keys, n_items, seed, indexed):
    """A burst of Blocks, Timeouts and TCs from test_groups_dev's generator, over this file's key array.  That generator signs with
    committee keys [0, its K) and foreign keys [its K, its K + its FOREIGN), so it shares this file's committee only while its K equals
    K and its FOREIGN is at most FOREIGN (test_group_generator_shares_this_files_keys checks both)."""
    from test_groups_dev import expected, make_burst
    b = make_burst(oracle, keys, np.random.default_rng(seed), n_items, foreign=not indexed)
    groups, items = expected(oracle, keys, b, indexed=indexed)
    if indexed:  # removed committee slots reject their items
        items = items & live_mask()[b["kidx"]]
        groups = np.ones(b["n_groups"], bool)
        np.logical_and.at(groups, b["gi"], items)
    return b, items, groups


@pytest.mark.gpu
@pytest.mark.parametrize("indexed", [False, True])
def test_groups_dev(s, committee, oracle, keys, indexed):
    from test_groups_dev import to_device
    b, items, groups = group_set(oracle, keys, 700, 800 + indexed, indexed)
    d = to_device(b, indexed=indexed)
    n, G = len(b["mi"]), b["n_groups"]
    d_sig, d_pre = garbage(d["sig"]), garbage(d["pre"], shift=True)
    ib, gb = bitmap(n), bitmap(G)
    land([(d_sig, d["sig"]), (d_pre, d["pre"])])
    committee.verify_groups_dev(d_pre, d["off"], len(b["off"]) - 1, d_sig, d["mi"], ib, n, d_mode=d["mode"], d_pk=d["pk"], d_vidx=d["vidx"])
    committee.qc_and_dev(ib, d["gi"], n, G, gb)
    s.synchronize()
    check_bitmap(ib, items, "verify_groups_dev items indexed=%s" % indexed)
    check_bitmap(gb, groups, "qc_and_dev groups indexed=%s" % indexed)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097])
def test_keygen_and_sign_dev(s, engine, oracle, n):
    torch = _torch()
    rng = np.random.default_rng(900 + n)
    seeds = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    n_sig = n + 7
    kidx = rng.integers(0, n, n_sig).astype(np.uint32)
    dg = rng.integers(0, 256, (n_sig, 32), dtype=np.uint8)
    want_own = oracle.sign_batch(seeds, pks, np.arange(n, dtype=np.uint32), dg[:n].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    want_idx = oracle.sign_batch(seeds, pks, kidx, dg.reshape(-1), np.arange(n_sig + 1, dtype=np.uint64) * 32)
    src_seeds, src_dg, d_pks, d_kidx = dev(seeds), dev(dg), dev(pks), dev(kidx)
    d_seeds, d_dg = garbage(src_seeds), garbage(src_dg, shift=True)
    out_pk = torch.full((n, 32), 0xA5, dtype=torch.uint8, device="cuda")
    out_own = torch.full((n, 64), 0xA5, dtype=torch.uint8, device="cuda")
    out_idx = torch.full((n_sig, 64), 0xA5, dtype=torch.uint8, device="cuda")
    land([(d_seeds, src_seeds), (d_dg, src_dg)])
    engine.keygen_batch_dev(d_seeds, out_pk, n)
    engine.sign_digests_dev(d_seeds, d_pks, n, d_dg, out_own, n)
    engine.sign_digests_dev(d_seeds, d_pks, n, d_dg, out_idx, n_sig, d_key_idx=d_kidx)
    s.synchronize()
    assert np.array_equal(out_pk.cpu().numpy(), pks), "keygen_batch_dev differs from the oracle"
    assert np.array_equal(out_own.cpu().numpy(), want_own), "sign_digests_dev (key i) differs from the oracle"
    assert np.array_equal(out_idx.cpu().numpy(), want_idx), "sign_digests_dev (key_idx) differs from the oracle"


@pytest.mark.gpu
def test_empty_calls_leave_outputs_alone(s, committee):
    torch = _torch()
    e = committee
    u8 = torch.zeros(256, dtype=torch.uint8, device="cuda")
    i32 = torch.zeros(8, dtype=torch.int32, device="cuda")
    i64 = torch.zeros(8, dtype=torch.int64, device="cuda")
    outs = {}

    def out(name):
        outs[name] = bitmap(64)
        return outs[name]

    e.verify_rec128_dev(u8, out("rec128"), 0)
    e.verify_var_dev(u8, u8, u8, i64, out("var"), 0)
    e.verify_committee_dev(i32, u8, u8, out("committee"), 0)
    e.verify_committee_dev(i32, u8, u8, out("committee midx"), 0, d_midx=i32)
    e.verify_msgs_dev(u8, u8, 32, out("msgs digests"), out("msgs"), 0, d_pk=u8)
    e.verify_msgs_dev(u8, u8, 32, out("msgs vidx digests"), out("msgs vidx"), 0, d_vidx=i32)
    e.digest32_dev(u8, i64, out("digest32"), 0)
    e.digest32_fixed_dev(u8, 40, out("digest32_fixed"), 0)
    e.verify_qc_votes_dev(u8, u8, i32, out("qc votes"), 0, d_pk=u8)
    e.verify_qc_votes_dev(u8, u8, i32, out("qc votes vidx"), 0, d_vidx=i32)
    e.qc_and_dev(i32, i32, 0, 0, out("qc_and"))
    e.verify_groups_dev(u8, i64, 0, u8, i32, out("groups"), 0, d_pk=u8)
    e.keygen_batch_dev(u8, out("keygen"), 0)
    e.sign_digests_dev(u8, u8, 1, u8, out("sign"), 0)
    e.sign_digests_dev(u8, u8, 1, u8, out("sign key_idx"), 0, d_key_idx=i32)
    s.synchronize()
    for name, t in outs.items():
        untouched(t, name)


# ---------------------------------------------------------------------------------------------------- engine state on the caller's stream
@pytest.mark.gpu
def test_key_cache_learns_on_the_callers_stream(s, oracle, keys):
    """No committee, 40 distinct keys: the first pass parks keys 0..19, the second builds their tables on the caller's stream and parks
    20..39, the third builds those.  A host call straight after the third pass reads the tables built on the caller's stream."""
    e = fresh_engine()
    try:
        sets = [rec_set(oracle, keys, n, seed=1000 + n, key_hi=hi, adversarial=False) for n, hi in ((500, 20), (700, 40), (900, 40))]
        outs = []
        for j, recs in enumerate(sets):
            src = dev(recs)
            d = garbage(src)  # zero keys: a pass that learned from them before the copy would cache the wrong key
            bm = bitmap(len(recs))
            land([(d, src)])
            e.verify_rec128_dev(d, bm, len(recs), 0)
            outs.append((bm, src, d))
            if j < 2:
                s.synchronize()
                assert e.cached_keys == 20 * j, "after pass %d: %d keys cached" % (j + 1, e.cached_keys)
        assert e.cached_keys == 40
        host = rec_set(oracle, keys, 200, seed=1999, key_lo=20, key_hi=40, adversarial=False)
        got_host = e.verify_rec128(host)
        s.synchronize()
        for j, (bm, _, _) in enumerate(outs):
            check_bitmap(bm, oracle.verify_rec128(sets[j], 0), "learning pass %d" % (j + 1))
        assert np.array_equal(got_host, oracle.verify_rec128(host, 0)), "host call after the learning passes differs from the oracle"
    finally:
        e.close()


@pytest.mark.gpu
def test_deferred_mode_across_every_verify_call(s, oracle, keys):
    """Twelve back-to-back deferred passes rotating through the five verify calls, each larger than the last, so both scratch sets grow
    while the other set's tail is in flight; every bitmap equals the oracle after results_wait."""
    from test_groups_dev import to_device
    torch = _torch()
    e = fresh_engine(keys)
    try:
        ns = [40, 90, 200, 400, 700, 1100, 1600, 2300, 3100, 4200, 5600, 7300]
        kinds = ["rec128", "var", "committee", "msgs", "groups"]
        plans = []
        for j, n in enumerate(ns):
            rng = np.random.default_rng(1100 + j)
            kind = kinds[j % len(kinds)]
            if kind == "rec128":
                recs = rec_set(oracle, keys, n, seed=1100 + j)
                plans.append((kind, n, dict(d=dev(recs)), oracle.verify_rec128(recs, 1), 1))
            elif kind == "var":
                sig, pk, msgs, off = var_set(oracle, keys, rng, list(rng.integers(0, 301, max(1, n // 12))), reps=1)
                n = sig.shape[0]
                plans.append((kind, n, dict(sig=dev(sig), pk=dev(pk), msgs=dev(np.append(msgs, np.uint8(0))), off=dev(off)),
                              oracle.verify_var(sig, pk, msgs, off, mode=0), 0))
            elif kind == "committee":
                vidx = rng.integers(0, K, n).astype(np.uint32)
                dg = rng.integers(0, 256, (3, 32), dtype=np.uint8)
                midx = rng.integers(0, 3, n).astype(np.uint32)
                sig = sign_digests(oracle, keys, vidx, dg[midx], rng)
                want = oracle.verify_rec128(np.concatenate([sig, keys[1][vidx], dg[midx]], axis=1), 0)
                plans.append((kind, n, dict(vidx=dev(vidx), sig=dev(sig), dg=dev(dg), midx=dev(midx)), want, 0))
            elif kind == "msgs":
                msgs = rng.integers(0, 256, (n, 64), dtype=np.uint8)
                kidx = rng.integers(0, K, n).astype(np.uint32)
                dg = np.array([digest(m) for m in msgs])
                sig = sign_digests(oracle, keys, kidx, dg, rng)
                want = oracle.verify_rec128(np.concatenate([sig, keys[1][kidx], dg], axis=1), 1)
                plans.append((kind, n, dict(sig=dev(sig), msgs=dev(msgs), pk=dev(keys[1][kidx]),
                                            dig=torch.empty((n, 32), dtype=torch.uint8, device="cuda")), want, 1))
            else:
                b, items, _ = group_set(oracle, keys, n, 1100 + j, False)
                plans.append((kind, n, dict(b=b, d=to_device(b)), items, None))
        s.synchronize()
        e.set_deferred(True)
        bms = []
        for kind, n, d, _, mode in plans:
            bm = bitmap(n)
            bms.append(bm)
            if kind == "rec128":
                e.verify_rec128_dev(d["d"], bm, n, mode)
            elif kind == "var":
                e.verify_var_dev(d["sig"], d["pk"], d["msgs"], d["off"], bm, n, mode)
            elif kind == "committee":
                e.verify_committee_dev(d["vidx"], d["sig"], d["dg"], bm, n, d_midx=d["midx"], mode=mode)
            elif kind == "msgs":
                e.verify_msgs_dev(d["sig"], d["msgs"], 64, d["dig"], bm, n, d_pk=d["pk"], mode=mode)
            else:
                b, g = d["b"], d["d"]
                e.verify_groups_dev(g["pre"], g["off"], len(b["off"]) - 1, g["sig"], g["mi"], bm, n, d_mode=g["mode"], d_pk=g["pk"])
        e.results_wait()
        s.synchronize()
        e.set_deferred(False)
        for (kind, n, _, want, _), bm in zip(plans, bms):
            check_bitmap(bm, want, "deferred %s n=%d" % (kind, n))
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------------- host calls after a `_dev` pass
def _latency_recs(oracle, keys, seed):
    """40 records of registered, live keys: hs_verify_rec128 takes the latency path (64 records or fewer)."""
    rng = np.random.default_rng(seed)
    kidx = (np.arange(40) + 10).astype(np.uint32)
    msgs = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    return np.concatenate([sign_digests(oracle, keys, kidx, msgs, rng, corrupt=0.1), keys[1][kidx], msgs], axis=1)


def _warm(e, oracle, keys):
    """One host call of 2^20 records, so every scratch buffer the next calls use is large enough and none of them synchronises the
    device to grow one; and one latency-path call, so its kernel is loaded (a first launch may load the module, which can wait for
    the device)."""
    recs, want = tiled(oracle, keys, BIG, seed=31, adversarial=False)
    assert np.array_equal(e.verify_rec128(recs), want)
    small = _latency_recs(oracle, keys, 30)
    assert np.array_equal(e.verify_rec128(small), oracle.verify_rec128(small, 0))


def _committee_pass(oracle, keys, n, seed):
    vidx, midx, digests, sig, strict, _ = committee_set(oracle, keys, n, np.random.default_rng(seed), 5)
    return dict(vidx=dev(vidx), midx=dev(midx), dg=dev(digests), sig=dev(sig)), strict


@pytest.mark.gpu
def test_host_call_waits_for_the_dev_pass_that_owns_the_scratch(s, oracle, keys):
    e = fresh_engine(keys, remove=REMOVED)
    try:
        _warm(e, oracle, keys)
        d, want = _committee_pass(oracle, keys, 4096, 1200)
        host = rec_set(oracle, keys, 5000, seed=1201, adversarial=False)
        bm = bitmap(4096)
        s.synchronize()
        _torch().cuda._sleep(LONG_SLEEP)
        e.verify_committee_dev(d["vidx"], d["sig"], d["dg"], bm, 4096, d_midx=d["midx"])
        got = e.verify_rec128(host)
        done = s.query()
        s.synchronize()
        assert done, "the host call returned while the _dev pass it shares scratch with was still queued"
        check_bitmap(bm, want, "verify_committee_dev before a host call")
        assert np.array_equal(got, oracle.verify_rec128(host, 0)), "host call after a _dev pass differs from the oracle"
    finally:
        e.close()


@pytest.mark.gpu
def test_latency_path_does_not_wait_for_a_dev_pass(s, oracle, keys):
    e = fresh_engine(keys, remove=REMOVED)
    try:
        _warm(e, oracle, keys)
        d, want = _committee_pass(oracle, keys, 4096, 1300)
        host = _latency_recs(oracle, keys, 1301)
        s.synchronize()
        bm = bitmap(4096)
        _torch().cuda._sleep(LONG_SLEEP)
        e.verify_committee_dev(d["vidx"], d["sig"], d["dg"], bm, 4096, d_midx=d["midx"])
        got = e.verify_rec128(host)
        done = s.query()
        s.synchronize()
        assert not done, "the latency path waited for a _dev pass it shares no scratch with"
        check_bitmap(bm, want, "verify_committee_dev beside the latency path")
        assert np.array_equal(got, oracle.verify_rec128(host, 0)), "latency path beside a _dev pass differs from the oracle"
    finally:
        e.close()


@pytest.mark.gpu
def test_table_audit_does_not_wait_for_a_dev_pass(s, oracle, keys):
    """The audit stages on its own stream into its own scratch (as the scrub's ticks and the slot builds of repairs and staged changes
    do), so it neither waits for a _dev pass nor queues behind one."""
    e = fresh_engine(keys, remove=REMOVED)
    try:
        _warm(e, oracle, keys)
        assert e.table_audit()[0] == 0  # creates the audit's stream and scratch, and loads its kernels
        d, want = _committee_pass(oracle, keys, 4096, 1500)
        s.synchronize()
        bm = bitmap(4096)
        _torch().cuda._sleep(LONG_SLEEP)
        e.verify_committee_dev(d["vidx"], d["sig"], d["dg"], bm, 4096, d_midx=d["midx"])
        failed, _ = e.table_audit()
        done = s.query()
        s.synchronize()
        assert not done, "the table audit waited for a _dev pass it shares no scratch with"
        assert failed == 0, "the audit found a fault in a clean context: %s" % e.last_error
        check_bitmap(bm, want, "verify_committee_dev beside a table audit")
    finally:
        e.close()


@pytest.mark.gpu
def test_host_call_overlapping_a_large_dev_pass(s, oracle, keys):
    """No sleep: a 2^20-record pass on the caller's stream, then at once a host call of 20,000 records over the same scratch rows."""
    e = fresh_engine(keys, remove=REMOVED)
    try:
        _warm(e, oracle, keys)
        recs, want = tiled(oracle, keys, BIG, seed=1400, adversarial=False)
        host = rec_set(oracle, keys, 20000, seed=1401, adversarial=False)
        src = dev(recs)
        bm = bitmap(BIG)
        s.synchronize()
        e.verify_rec128_dev(src, bm, BIG, 0)
        got = e.verify_rec128(host)
        s.synchronize()
        assert np.array_equal(got, oracle.verify_rec128(host, 0)), "host call beside a large _dev pass differs from the oracle"
        check_bitmap(bm, want, "verify_rec128_dev of 2^20 records beside a host call")
    finally:
        e.close()
