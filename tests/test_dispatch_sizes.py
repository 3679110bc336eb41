"""The synchronous throughput path at every size where its dispatch changes shape, bit for bit against the CPU oracle: the finish
kernel's records per thread (4, 8 or 16, chosen from the record count in run_verify) with ragged blocks, thread groups and bitmap
words; the generic side pass over the committee lookup's misses past the first iteration of its capped grid; the fixed-length Digest
at tails that need one or two blocks after the full ones, and from misaligned buffers; and the chunk seams of hs_verify_msgs.

Every threshold is read from hs_engine.cu, and a CPU test checks that each planned size sits on the side of each threshold it claims,
so moving a cut-over fails here instead of quietly testing another shape.

Expected verdicts at 2^19 records come without 2^19 oracle verifies: a base set, verified once by the oracle in both modes, is tiled
to the size, and sentinel positions get a bit flip in S or in the message and are re-verified by the oracle alone.  Sentinels sit at
the last two records, on both sides of every finish-block seam of each group width, at the last record of each thread's group in the
first and the last finish block, and at lane w % 32 of every bitmap word w, so a word written to the wrong index or shifted by one
group cannot go unseen."""
import hashlib
import os
import re

import numpy as np
import pytest

from oracle_api import L_ORDER, P, make_adversarial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC_PATH = os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")

# ---------------------------------------------------------------------------------------------------- thresholds from the source
PATTERNS = {
    "threads": r"#define HS_THREADS (\d+)\b",
    # run_verify: records per finish thread
    "finish": r"const int fin_group = \(defer \|\| n >= \(1u << (\d+)\)\) \? 16 : \(n >= \(1u << (\d+)\) \? 8 : 4\);",
    # launch_main: the generic pass over the lookup's misses, 32-thread blocks, grid capped at n_sms * 8
    "miss_grid": r"unsigned grid = blocks_for\(n, (\d+)\);\s*if \(grid > c->n_sms \* (\d+)u\) grid = c->n_sms \* \2u;\s*"
                 r"k_verify_main<false><<<grid, \1, 0, S\.side>>>\(L, 0, S\.miss_count, S\.miss,",
    # launch_digest_fixed: the staged kernel's conditions, and the constant padding block
    "digest_fixed": r"if \(msg_len >= (\d+) && \(msg_len & (\d+)\) == 0 && \(reinterpret_cast<uintptr_t>\(d_msgs\) & (\d+)\) == 0\) \{\s*"
                    r"sha512_kw kw;\s*const int pad_is_const = \(msg_len & (\d+)\) == 0;",
    # hs_verify_msgs: records per chunk, and HS_CHUNK_RECORDS's floor and rounding
    "chunk": r"size_t CH = 1u << (\d+);.{0,400}?if \(const char \*e = getenv\(\"HS_CHUNK_RECORDS\"\)\) \{\s*size_t v = strtoull\(e, nullptr, 10\);\s*"
             r"if \(v >= (\d+)\) CH = v & ~\(size_t\)(\d+);",
}


def thresholds():
    src = open(SRC_PATH).read()
    m = {k: re.search(p, src, re.S) for k, p in PATTERNS.items()}
    missing = [k for k, v in m.items() if v is None]
    assert not missing, "hs_engine.cu no longer matches %s: update the size plan of this file with the dispatch" % missing
    f, g, d, c = m["finish"], m["miss_grid"], m["digest_fixed"], m["chunk"]
    return dict(threads=int(m["threads"].group(1)), fin16=1 << int(f.group(1)), fin8=1 << int(f.group(2)),
                miss_threads=int(g.group(1)), miss_blocks_per_sm=int(g.group(2)),
                fixed_min=int(d.group(1)), fixed_mult=int(d.group(2)) + 1, fixed_align=int(d.group(3)) + 1, pad_const=int(d.group(4)) + 1,
                chunk_default=1 << int(c.group(1)), chunk_floor=int(c.group(2)), chunk_round=int(c.group(3)) + 1)


def fin_group(T, n):
    """Records per thread of the finish kernel for a non-deferred pass of n records (run_verify)."""
    return 16 if n >= T["fin16"] else (8 if n >= T["fin8"] else 4)


def digest_kernel(T, msg_len, aligned=True):
    """Which Digest launch_digest_fixed picks: the staged kernel with the constant padding block, the staged kernel with a tail, or
    the generic per-thread reader."""
    if msg_len >= T["fixed_min"] and msg_len % T["fixed_mult"] == 0 and aligned:
        return "fixed_const" if msg_len % T["pad_const"] == 0 else "fixed_tail"
    return "generic"


def chunk_records(T, env):
    """Records per chunk of hs_verify_msgs with HS_CHUNK_RECORDS = env (None: unset)."""
    v = int(env) if env is not None else 0
    return v & ~(T["chunk_round"] - 1) if v >= T["chunk_floor"] else T["chunk_default"]


# name -> (threshold, offset, records per finish thread): the last group-4 size, both ends of group 8, and group 16 at a multiple of
# a finish block and past it with a ragged block, thread group and word
FINISH_SIZES = {"last4": ("fin8", -1, 4), "first8": ("fin8", 0, 8), "ragged8": ("fin8", 1031, 8), "last8": ("fin16", -1, 8),
                "first16": ("fin16", 0, 16), "ragged16": ("fin16", 2048 + 13, 16)}
DIGEST_LENS = [16, 48, 96, 112, 128, 144, 224, 240, 256, 368, 496, 1008, 1136]
DIGEST_COUNTS = [1, 31, 32, 33, 129, 4097]
CHUNK_ENV, CHUNK_N_FULL, CHUNK_TAIL = "1100", 7, 33


def finish_size(T, name):
    th, off, _ = FINISH_SIZES[name]
    return T[th] + off


def miss_records(T, n_sms):
    """Misses of the side-pass test: three full grids of the capped side pass and 77 records into a fourth iteration."""
    return 3 * n_sms * T["miss_blocks_per_sm"] * T["miss_threads"] + 77


def miss_layout(m):
    """Positions of the side-pass test: two misses, then a record of a registered key, until there are m misses."""
    n = m + m // 2
    is_miss = (np.arange(n) % 3) != 2
    assert is_miss.sum() == m
    return is_miss


# ---------------------------------------------------------------------------------------------------- signed sets
IDENTITY = (1).to_bytes(32, "little")
ORDER2 = (P - 1).to_bytes(32, "little")
Y8 = 0x05fc536d880238b13933c6d305acdfd5f098eff289f4c345b027b2c28f95e826
TORSION = [int(y).to_bytes(32, "little") for y in (P - 1, Y8, P - Y8)] + [bytes(int(y).to_bytes(32, "little")[:31]) + b"\x80" for y in (Y8, P - Y8)]
B_ENC = int("6666666666666666666666666666666666666666666666666666666666666658", 16).to_bytes(32, "little")


def _digest(b):
    return hashlib.sha512(bytes(b)).digest()[:32]


def _secret(seed):
    h = hashlib.sha512(bytes(seed)).digest()
    return int.from_bytes(bytes([h[0] & 248]) + h[1:31] + bytes([(h[31] & 127) | 64]), "little"), h[32:]


def signed_set(oracle, rng, seeds, pks, n, msg_len=None, corrupt=0.03, n_adv=0):
    """n records over the Digests of their own preimages (msg_len bytes each, or 16..199), key i % len(pks), `corrupt` of them with a
    bit flip in the signature or the preimage (never the key, so each record stays on the key path it was built for); then n_adv
    records over further preimages with the keys where implementations disagree: R = the identity with S = k * a under an honest key
    (batch-eq accepts, strict rejects), a small-order key (identity or order 2, R = identity, S = 0), a mixed-order key A + T signed
    with a, and a key that does not decompress.  Returns dict(recs (n + n_adv, 128), pre: list of bytes)."""
    lens = np.full(n + n_adv, msg_len) if msg_len else rng.integers(16, 200, n + n_adv)
    pre = [rng.bytes(int(x)) for x in lens]
    kidx = (np.arange(n) % len(pks)).astype(np.uint32)
    dig = np.array([np.frombuffer(_digest(p), np.uint8) for p in pre[:n]])
    sig = oracle.sign_batch(seeds, pks, kidx, dig.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    recs = np.zeros((n + n_adv, 128), np.uint8)
    recs[:n, :64], recs[:n, 64:96] = sig, pks[kidx]
    for i in rng.choice(n, int(n * corrupt), replace=False):
        if rng.integers(2):
            recs[i, int(rng.integers(64))] ^= np.uint8(1 << int(rng.integers(8)))
        else:
            q = bytearray(pre[i])
            q[int(rng.integers(len(q)))] ^= 1 << int(rng.integers(8))
            pre[i] = bytes(q)
    for j in range(n, n + n_adv):
        k = int(rng.integers(len(pks)))
        a, prefix = _secret(seeds[k])
        A, m = pks[k].tobytes(), _digest(pre[j])
        kind = j % 4
        if kind == 0:                                   # R = identity, S = k * a: the cofactorless equation holds
            h = oracle.sc_reduce64(hashlib.sha512(IDENTITY + A + m).digest())
            sig = IDENTITY + (h * a % L_ORDER).to_bytes(32, "little")
        elif kind == 1:                                 # small-order key
            A, sig = (IDENTITY if rng.integers(2) else ORDER2), IDENTITY + bytes(32)
        elif kind == 2:                                 # mixed-order key A + T, signed with a
            A = oracle.point_add(A, TORSION[int(rng.integers(len(TORSION)))]) or A
            r = int.from_bytes(hashlib.sha512(prefix + m).digest(), "little") % L_ORDER
            R = oracle.scalarmult(r, B_ENC)
            h = oracle.sc_reduce64(hashlib.sha512(R + A + m).digest())
            sig = R + ((r + h * a) % L_ORDER).to_bytes(32, "little")
        else:                                           # a key that does not decompress, under an honest signature
            sig = oracle.sign(seeds[k].tobytes(), m)
            A = rng.bytes(32)
            while oracle.decompress_ok(A):
                A = rng.bytes(32)
        recs[j, :64], recs[j, 64:96] = np.frombuffer(sig, np.uint8), np.frombuffer(A, np.uint8)
    recs[:, 96:] = np.array([np.frombuffer(_digest(p), np.uint8) for p in pre])
    return dict(recs=recs, pre=pre)


def with_verdicts(oracle, recs, pre):
    """A base set: its records, their preimages (None where the message is not a preimage's Digest) and the oracle's verdicts."""
    return dict(recs=recs, pre=pre, strict=oracle.verify_rec128(recs, mode=0), eq=oracle.verify_rec128(recs, mode=1))


def concat(*sets):
    return dict(recs=np.concatenate([s["recs"] for s in sets]), pre=sum((list(s["pre"]) for s in sets), []))


def keys(seed, n):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------- sentinels
def sentinel_positions(T, n):
    """The records a finish or bitmap fault would get wrong first (see the module docstring)."""
    group = fin_group(T, n)
    pos = [np.array([n - 2, n - 1])]
    for g in (4, 8, 16):
        seams = np.arange(T["threads"] * g, n, T["threads"] * g)
        pos += [seams - 1, seams]
    block = T["threads"] * group
    for start in (0, (n - 1) // block * block):
        pos.append(np.arange(start + group - 1, min(n, start + block), group))
    w = np.arange((n + 31) // 32)
    pos.append(w * 32 + w % 32)
    p = np.unique(np.concatenate(pos))
    return p[(p >= 0) & (p < n)]


def arrange(oracle, base, src, sentinels):
    """Record i is base record src[i]; each sentinel p then gets a bit flip in S or in its message, chosen from p alone, and only the
    sentinels are re-verified by the oracle.  A message flip changes a byte of the preimage when the record has one (and its Digest with
    it), the message itself otherwise.  Returns recs, want_s, want_e, and pre / pre_idx: record i's message is the Digest of
    pre[pre_idx[i]] (for bases whose every record has a preimage)."""
    recs = base["recs"][src]
    pre = list(base["pre"])
    pre_idx = src.astype(np.uint32)
    for p in sentinels.tolist():
        h = (p * 0x9E3779B1) & 0xffffffff
        b = int(src[p])
        if (h >> 13) & 1:
            recs[p, 32 + (h & 31)] ^= np.uint8(1 << ((h >> 5) & 7))
        elif pre[b] is not None:
            q = bytearray(pre[b])
            q[h % len(q)] ^= 1 << ((h >> 8) & 7)
            pre_idx[p] = len(pre)
            pre.append(bytes(q))
            recs[p, 96:] = np.frombuffer(_digest(q), np.uint8)
        else:
            recs[p, 96 + (h & 31)] ^= np.uint8(1 << ((h >> 5) & 7))
    want_s, want_e = base["strict"][src], base["eq"][src]
    if sentinels.size:
        want_s[sentinels] = oracle.verify_rec128(recs[sentinels], mode=0)
        want_e[sentinels] = oracle.verify_rec128(recs[sentinels], mode=1)
    return dict(recs=recs, want_s=want_s, want_e=want_e, pre=pre, pre_idx=pre_idx)


def item_modes(n):
    """Per-item verdict modes, strict and batch-eq in turn with a period (6) that lines up with no thread group or bitmap word."""
    return ((np.arange(n) % 6) >= 3).astype(np.uint8)


def group_of(n):
    """Items into groups of 3 (certificates that straddle thread groups and words, small enough that many hold no rejected item), and
    one empty group at the end."""
    return (np.arange(n) // 3).astype(np.uint32), (n + 2) // 3 + 1


def groups_form(A):
    """verify_groups arrays of an arrangement whose every record has a preimage: the preimages, their offsets and the expectations of
    each item in its mode and of each group's AND."""
    pre = np.frombuffer(b"".join(A["pre"]), np.uint8)
    off = np.zeros(len(A["pre"]) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in A["pre"]])
    n = A["recs"].shape[0]
    modes = item_modes(n)
    gi, n_groups = group_of(n)
    items = np.where(modes == 1, A["want_e"], A["want_s"])
    groups = np.ones(n_groups, bool)
    np.logical_and.at(groups, gi, items)
    return dict(pre=pre, off=off, modes=modes, gi=gi, n_groups=n_groups, items=items, groups=groups)


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def finish_base(oracle):
    """4,096 honest records over 64 keys (3 % corrupted) and 512 records with adversarial keys, all over preimage Digests (the
    verify_groups base), then 1,000 make_adversarial records (the rec128 / committee base)."""
    rng = np.random.default_rng(2024)
    seeds = keys(2025, 64)
    pks = oracle.keygen_batch(seeds)
    d = signed_set(oracle, rng, seeds, pks, 4096, n_adv=512)
    digest_only = with_verdicts(oracle, d["recs"], d["pre"])
    adv = make_adversarial(oracle, 1000, seed=2026)
    full = with_verdicts(oracle, np.concatenate([d["recs"], adv]), d["pre"] + [None] * len(adv))
    return dict(full=full, digest_only=digest_only)


TABLE_BUDGET = 4 << 30  # the tests' committees need no wide comb windows: a few GB of tables, not most of a shared device


def _register(engine, pks):
    engine.set_table_budget(TABLE_BUDGET)
    return engine.committee_register(pks)


def _clear(engine):
    """No committee, an empty key cache, and the table budget the context started with."""
    engine.committee_register(np.zeros((0, 32), np.uint8))
    engine.set_table_budget(int(os.environ.get("HS_TABLE_BUDGET_MB", "0")) << 20)


def _register_unique(engine, recs):
    """Registers every distinct key of recs; returns each record's committee index."""
    ukeys, inv = np.unique(recs[:, 64:96], axis=0, return_inverse=True)
    _register(engine, ukeys)
    return inv.reshape(-1).astype(np.uint32)


def _first_bad(got, want):
    return np.flatnonzero(got != want)[:10]


# ---------------------------------------------------------------------------------------------------- CPU
def test_thresholds_and_size_plan():
    """The dispatch thresholds still parse from hs_engine.cu, and every size this file runs sits where it claims."""
    T = thresholds()
    assert T["threads"] == 128 and T["fin8"] < T["fin16"]
    for name, (_, _, g) in FINISH_SIZES.items():
        n = finish_size(T, name)
        assert fin_group(T, n) == g, (name, n)
        if name.startswith(("ragged", "last")):  # a partial finish block, thread group and bitmap word
            assert n % (T["threads"] * g) and n % g and n % 32, (name, n)
    assert {fin_group(T, finish_size(T, k)) for k in FINISH_SIZES} == {4, 8, 16}
    # the side pass: 3 full capped grids and a fourth iteration, on any H100 (114 SMs on PCIe, 132 on SXM)
    for n_sms in (114, 132):
        m = miss_records(T, n_sms)
        grid_threads = n_sms * T["miss_blocks_per_sm"] * T["miss_threads"]
        assert -(-m // T["miss_threads"]) > n_sms * T["miss_blocks_per_sm"]  # the cap binds
        assert -(-m // grid_threads) == 4
        is_miss = miss_layout(m)
        # hs_verify_msgs splits the call into chunks: its first chunk alone still needs three iterations of the side pass
        assert is_miss.size > T["chunk_default"] and is_miss[:T["chunk_default"]].sum() > 2 * grid_threads
    # the Digest: generic reader below one block, constant padding block, a tail that fits the last block, one that needs two
    kinds = {L: digest_kernel(T, L) for L in DIGEST_LENS}
    assert all(kinds[L] == "generic" for L in DIGEST_LENS if L < T["fixed_min"])
    assert [L for L in DIGEST_LENS if kinds[L] == "fixed_const"] == [128, 256]
    two_more = [L for L in DIGEST_LENS if kinds[L] == "fixed_tail" and (L + 17 + 127) // 128 - L // 128 == 2]
    one_more = [L for L in DIGEST_LENS if kinds[L] == "fixed_tail" and (L + 17 + 127) // 128 - L // 128 == 1]
    assert two_more == [240, 368, 496, 1008, 1136] and one_more == [144, 224]
    assert all(digest_kernel(T, L, aligned=False) == "generic" for L in DIGEST_LENS)
    assert digest_kernel(T, 240) == "fixed_tail" and digest_kernel(T, 368) == "fixed_tail" and digest_kernel(T, 100) == "generic"
    # chunk seams: HS_CHUNK_RECORDS rounds down to a multiple of 32 and is ignored below its floor
    assert chunk_records(T, None) == T["chunk_default"] == 1 << 17
    ch = chunk_records(T, CHUNK_ENV)
    assert ch == 1088 and T["chunk_floor"] == 1024
    assert chunk_records(T, str(T["chunk_floor"] - 1)) == T["chunk_default"]
    n = CHUNK_N_FULL * ch + CHUNK_TAIL
    assert -(-n // ch) == CHUNK_N_FULL + 1 and -(-n // int(CHUNK_ENV)) == CHUNK_N_FULL  # the rounding shows in the chunk count
    assert n < T["chunk_default"]


def test_sentinel_expectations_equal_the_oracle(oracle):
    """On a small tiled case the builder's expectations equal the oracle on every record, in both modes, and for verify_groups the
    preimage list reproduces every record's message."""
    T = thresholds()
    rng = np.random.default_rng(7)
    seeds = keys(8, 8)
    pks = oracle.keygen_batch(seeds)
    d = signed_set(oracle, rng, seeds, pks, 200, n_adv=48)
    adv = make_adversarial(oracle, 60, seed=9)
    base = with_verdicts(oracle, np.concatenate([d["recs"], adv]), d["pre"] + [None] * 60)
    assert (base["strict"] != base["eq"]).sum() >= 10 and base["strict"].sum() > 100
    n = 3001
    sent = sentinel_positions(T, n)
    assert {0, n - 2, n - 1, 511, 512, 1023, 1024, 2047, 2048, 3} <= set(sent.tolist())
    assert len({int(p) // 32 for p in sent}) == (n + 31) // 32
    src = np.arange(n) % base["recs"].shape[0]
    A = arrange(oracle, base, src, sent)
    assert (A["want_s"] == oracle.verify_rec128(A["recs"], mode=0)).all()
    assert (A["want_e"] == oracle.verify_rec128(A["recs"], mode=1)).all()
    assert (A["want_s"][sent] != base["strict"][src[sent]]).sum() > sent.size // 3  # the flips change verdicts
    # verify_groups form: digest-only base
    dbase = with_verdicts(oracle, d["recs"], d["pre"])
    src = np.arange(n) % dbase["recs"].shape[0]
    A = arrange(oracle, dbase, src, sent)
    G = groups_form(A)
    msgs = np.array([np.frombuffer(_digest(G["pre"][int(G["off"][j]):int(G["off"][j + 1])]), np.uint8) for j in A["pre_idx"]])
    assert (msgs == A["recs"][:, 96:]).all()
    assert (G["items"] == np.where(G["modes"] == 1, oracle.verify_rec128(A["recs"], mode=1), oracle.verify_rec128(A["recs"], mode=0))).all()
    assert G["groups"][-1] and not G["groups"].all()


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("size", list(FINISH_SIZES))
def test_finish_groups_rec128_and_committee(engine, oracle, finish_base, size):
    """The finish kernel at 4, 8 and 16 records per thread, at both ends of each width: verify_rec128 without a committee (generic
    main), with every base key registered (lookup, committee main), and verify_committee with msg_idx, in both modes."""
    T = thresholds()
    n = finish_size(T, size)
    base = finish_base["full"]
    assert (base["strict"] != base["eq"]).sum() >= 100
    src = np.arange(n) % base["recs"].shape[0]
    A = arrange(oracle, base, src, sentinel_positions(T, n))
    recs = A["recs"]
    try:
        for mode, want in ((0, A["want_s"]), (1, A["want_e"])):
            _clear(engine)  # no committee and an empty key cache: the generic main kernel over every record
            assert engine.cached_keys == 0
            got = engine.verify_rec128(recs, mode=mode)
            assert (got == want).all(), ("generic", mode, _first_bad(got, want))
        vidx = _register_unique(engine, base["recs"])[src]
        for mode, want in ((0, A["want_s"]), (1, A["want_e"])):
            got = engine.verify_rec128(recs, mode=mode)
            assert (got == want).all(), ("lookup", mode, _first_bad(got, want))
            got = engine.verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(n, dtype=np.uint32), mode=mode)
            assert (got == want).all(), ("indexed", mode, _first_bad(got, want))
    finally:
        _clear(engine)


@pytest.mark.gpu
@pytest.mark.parametrize("size", list(FINISH_SIZES))
def test_finish_groups_per_item_modes(engine, oracle, finish_base, size):
    """k_verify_finish_modes at every width: verify_groups with mode bytes that alternate strict and batch-eq out of step with the
    thread groups, over GPU-hashed preimages with a registered committee; item bits and group ANDs equal the oracle."""
    T = thresholds()
    n = finish_size(T, size)
    base = finish_base["digest_only"]
    src = np.arange(n) % base["recs"].shape[0]
    A = arrange(oracle, base, src, sentinel_positions(T, n))
    G = groups_form(A)
    recs = A["recs"]
    split = A["want_s"] != A["want_e"]
    assert (split & (G["modes"] == 0)).sum() > 1000 and (split & (G["modes"] == 1)).sum() > 1000
    try:
        _register_unique(engine, base["recs"])
        groups, items = engine.verify_groups(G["pre"], G["off"], recs[:, :64], A["pre_idx"], G["gi"], G["n_groups"], mode=G["modes"],
                                             pk=recs[:, 64:96], want_items=True)
        assert (items == G["items"]).all(), _first_bad(items, G["items"])
        assert (groups == G["groups"]).all(), _first_bad(groups, G["groups"])
        assert groups[-1] and not groups.all()
    finally:
        _clear(engine)


def build_miss_case(oracle, n_sms):
    """Records of 64 registered keys interleaved with records whose keys are not registered (honest keys, mixed-order, small-order
    and non-decompressible keys) over 48-byte preimages, with a sentinel flip on every 97th record."""
    T = thresholds()
    m = miss_records(T, n_sms)
    is_miss = miss_layout(m)
    rng = np.random.default_rng(3030)
    reg_seeds, out_seeds = keys(3031, 64), keys(3032, 64)
    reg_pks, out_pks = oracle.keygen_batch(reg_seeds), oracle.keygen_batch(out_seeds)
    hit = signed_set(oracle, rng, reg_seeds, reg_pks, 1500, msg_len=48)
    out = signed_set(oracle, rng, out_seeds, out_pks, 2000, msg_len=48, n_adv=600)
    base = with_verdicts(oracle, *concat(hit, out).values())
    n_hit = hit["recs"].shape[0]
    src = np.where(is_miss, n_hit + np.cumsum(is_miss) % out["recs"].shape[0], np.cumsum(~is_miss) % n_hit)
    A = arrange(oracle, base, src, np.arange(5, is_miss.size, 97))
    A["pre"] = np.frombuffer(b"".join(A["pre"]), np.uint8).reshape(-1, 48)[A["pre_idx"]]
    A.update(is_miss=is_miss, reg_pks=reg_pks)
    return A


@pytest.fixture(scope="module")
def miss_case(oracle):
    import torch
    return build_miss_case(oracle, torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.mark.gpu
def test_miss_pass_past_its_grid(engine, oracle, miss_case):
    """More misses than three full grids of the capped side pass: every grid-stride iteration of k_verify_main<false> over the compacted
    miss list, through verify_rec128, verify_var and verify_msgs with key bytes, in both modes.  A pass of rejected records first leaves
    the scratch holding rejections, so a miss the side pass skipped could not borrow an earlier verdict."""
    A = miss_case
    recs, n = A["recs"], A["recs"].shape[0]
    sig, pk, dig = recs[:, :64].copy(), recs[:, 64:96].copy(), recs[:, 96:].copy()
    reg = {bytes(k) for k in A["reg_pks"]}
    assert all((bytes(k) in reg) != miss for k, miss in zip(pk, A["is_miss"]))
    assert A["want_s"][A["is_miss"]].sum() > 1000 and (A["want_s"] != A["want_e"]).sum() > 100
    try:
        assert _register(engine, A["reg_pks"]).all()
        poisoned = recs.copy()
        poisoned[:, 63] |= 0xE0  # S >= 2^253: every record rejected
        assert not engine.verify_rec128(poisoned).any()
        assert engine.cached_keys == 0  # an explicit committee: unregistered keys stay on the miss pass, nothing is learned
        before = engine.kernel_launches
        got = engine.verify_rec128(recs, mode=0)
        assert engine.kernel_launches - before == 4  # lookup, side pass, committee main, finish
        assert (got == A["want_s"]).all(), _first_bad(got, A["want_s"])
        got = engine.verify_rec128(recs, mode=1)
        assert (got == A["want_e"]).all(), _first_bad(got, A["want_e"])
        off = np.arange(n + 1, dtype=np.uint64) * 32
        for mode, want in ((0, A["want_s"]), (1, A["want_e"])):
            got = engine.verify_var(sig, pk, dig.reshape(-1), off, mode=mode)
            assert (got == want).all(), ("var", mode, _first_bad(got, want))
            got = engine.verify_msgs(sig, A["pre"].reshape(-1), 48, pk=pk, mode=mode)
            assert (got == want).all(), ("msgs", mode, _first_bad(got, want))
        assert engine.cached_keys == 0
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_digest32_fixed_tails_and_misaligned_buffers(engine):
    """digest32_fixed_dev against hashlib at every length class (below one block, a tail that fits the last block, one that needs two
    more, a multiple of 128) and at counts around a warp and a block, from an aligned buffer and from views 4 and 8 bytes in."""
    import torch
    rng = np.random.default_rng(4040)
    for L in DIGEST_LENS:
        for n in DIGEST_COUNTS:
            data = rng.integers(0, 256, n * L, dtype=np.uint8)
            want = np.array([np.frombuffer(_digest(data[i * L:(i + 1) * L]), np.uint8) for i in range(n)])
            buf = torch.zeros(n * L + 16, dtype=torch.uint8, device="cuda")
            for shift in (0, 4, 8):
                view = buf[shift:shift + n * L]
                view.copy_(torch.from_numpy(data))
                out = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
                assert view.data_ptr() % 16 == shift
                engine.digest32_fixed_dev(view, L, out, n)
                got = out.cpu().numpy()
                assert (got == want).all(), (L, n, shift, np.flatnonzero((got != want).any(1))[:8])


def _msgs_set(oracle, seed, n, L, n_keys=64):
    """n records over L-byte messages (the signed message is their Digest), key i % n_keys, 5 % with a flipped signature bit."""
    rng = np.random.default_rng(seed)
    seeds = keys(seed + 1, n_keys)
    pks = oracle.keygen_batch(seeds)
    kidx = (np.arange(n) % n_keys).astype(np.uint32)
    msgs = rng.integers(0, 256, (n, L), dtype=np.uint8)
    dig = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
    sig = oracle.sign_batch(seeds, pks, kidx, dig.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    bad = rng.choice(n, n // 20, replace=False)
    sig[bad, rng.integers(0, 64, bad.size)] ^= np.uint8(0x10)
    return dict(sig=sig, msgs=msgs, dig=dig, kidx=kidx, pks=pks)


def _want(oracle, w, sig=None):
    recs = np.concatenate([w["sig"] if sig is None else sig, w["pks"][w["kidx"]], w["dig"]], axis=1)
    return oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [240, 368])
def test_verify_msgs_digest_tails(engine, oracle, L):
    """verify_msgs at lengths whose Digest tail needs two blocks after the full ones, with key bytes (no committee) and with validator
    indices, in both modes."""
    w = _msgs_set(oracle, 5000 + L, 2 * 1024 + 77, L)
    want = _want(oracle, w)
    assert (~want[0]).sum() >= 50
    pk = w["pks"][w["kidx"]]
    try:
        _clear(engine)
        for mode in (0, 1):
            got = engine.verify_msgs(w["sig"], w["msgs"].reshape(-1), L, pk=pk, mode=mode)
            assert (got == want[mode]).all(), ("pk", mode, _first_bad(got, want[mode]))
        assert _register(engine, w["pks"]).all()
        for mode in (0, 1):
            got = engine.verify_msgs(w["sig"], w["msgs"].reshape(-1), L, validator_idx=w["kidx"], mode=mode)
            assert (got == want[mode]).all(), ("validator_idx", mode, _first_bad(got, want[mode]))
    finally:
        _clear(engine)


@pytest.mark.gpu
@pytest.mark.parametrize("L", [240, 100])
def test_verify_msgs_chunk_seams(engine, oracle, monkeypatch, L):
    """HS_CHUNK_RECORDS = 1100 (1,088 records per chunk): 8 chunks, so both staging buffers are reused several times, and with half the
    signers registered every chunk runs the lookup and the side pass.  The first and last record of every chunk carry a flipped
    signature bit.  Verdicts equal the oracle and the one-chunk call, and a value below the floor is ignored."""
    T = thresholds()
    ch = chunk_records(T, CHUNK_ENV)
    n = CHUNK_N_FULL * ch + CHUNK_TAIL
    w = _msgs_set(oracle, 6000 + L, n, L)
    edges = np.unique(np.concatenate([np.arange(0, n, ch), np.minimum(np.arange(ch, n + ch, ch), n) - 1]))
    sig = w["sig"].copy()
    sig[edges, 40] ^= np.uint8(0x01)
    want = _want(oracle, w, sig)
    assert not want[0][edges].any()
    pk = w["pks"][w["kidx"]]
    assert (w["kidx"][:ch] >= 32).any() and (w["kidx"][-CHUNK_TAIL:] >= 32).any()
    launches = {}
    try:
        assert _register(engine, w["pks"][:32]).all()  # signers 32..63 are misses in every chunk
        for env in (CHUNK_ENV, str(T["chunk_floor"] - 1), None):
            if env is None:
                monkeypatch.delenv("HS_CHUNK_RECORDS", raising=False)
            else:
                monkeypatch.setenv("HS_CHUNK_RECORDS", env)
            for mode in (0, 1):
                before = engine.kernel_launches
                got = engine.verify_msgs(sig, w["msgs"].reshape(-1), L, pk=pk, mode=mode)
                launches[env] = engine.kernel_launches - before
                assert (got == want[mode]).all(), (env, mode, _first_bad(got, want[mode]))
        # Digest, lookup, side pass, committee main and finish per chunk
        assert launches == {CHUNK_ENV: 5 * -(-n // ch), str(T["chunk_floor"] - 1): 5, None: 5}
    finally:
        _clear(engine)
