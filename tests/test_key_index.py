"""key_index.h: the key -> slot index of the per-key comb tables, built on the host and probed by k_key_lookup.

CPU (tests/hostemu/key_index_emu.cpp, compiled by this module): on seeded random key sets with duplicated keys, the tables build() makes,
the slots find() returns under both accept rules the engine uses, and a sequence of insert_absent() calls equal a short restatement of
linear probing over key_hash here.
GPU: hs_committee_update gives a key added twice in one call one slot, also when the same call removed it."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_KEY = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------- the restatement
def key_hash(key):
    h = 0x9E3779B9
    for i in range(8):
        h ^= int.from_bytes(key[4 * i:4 * i + 4], "little")
        h = (h * 0x85EBCA6B) & 0xFFFFFFFF
        h ^= h >> 15
    return h


def capacity(n_slots):
    cap = 16
    while cap < 2 * n_slots:
        cap <<= 1
    return cap


def ref_probe(table, pks, key, accept):
    """(hash slot, key slot) of the first accepted key slot with these bytes on key's probe path, else (first empty hash slot, None)."""
    mask = len(table) - 1
    h = key_hash(key) & mask
    for _ in range(len(table)):
        if table[h] == NO_KEY:
            return h, None
        if accept(table[h]) and pks[table[h]] == key:
            return h, table[h]
        h = (h + 1) & mask
    return None, None


def ref_insert_absent(table, pks, idx, accept=lambda s: True):
    h, found = ref_probe(table, pks, pks[idx], accept)
    if found is not None:
        return False
    table[h] = idx
    return True


def ref_build(pks, n_slots, in_service):
    table = [NO_KEY] * capacity(n_slots)
    for i, keep in enumerate(in_service):
        if keep:
            ref_insert_absent(table, pks, i)
    return table


def ref_find(table, pks, key, accept):
    found = ref_probe(table, pks, key, accept)[1]
    return NO_KEY if found is None else found


# ---------------------------------------------------------------------------------------------------- the host build
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("keyindex") / "libhs_keyindex.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", lib, os.path.join(ROOT, "tests", "hostemu", "key_index_emu.cpp")])
    lib = ctypes.CDLL(lib)
    lib.emu_capacity.restype = ctypes.c_uint32
    lib.emu_capacity.argtypes = [ctypes.c_size_t]
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _blob(pks):
    return np.frombuffer(b"".join(pks), np.uint8).copy() if pks else np.zeros(32, np.uint8)


def emu_build(emu, pks, n_slots, in_service):
    out = np.zeros(emu.emu_capacity(n_slots), np.uint32)
    mask = np.array(in_service, np.uint8) if len(in_service) else np.zeros(1, np.uint8)
    emu.emu_build(_ptr(_blob(pks)), ctypes.c_size_t(len(pks)), ctypes.c_size_t(n_slots), _ptr(mask), _ptr(out))
    return out


def emu_find(emu, table, pks, keys, bound=None, accepted=None):
    t = np.array(table, np.uint32)
    out = np.zeros(len(keys), np.uint32)
    acc = None if accepted is None else np.array(accepted, np.uint8)
    emu.emu_find(_ptr(t), ctypes.c_uint32(len(t)), _ptr(_blob(pks)), _ptr(_blob(keys)), ctypes.c_size_t(len(keys)),
                 ctypes.c_uint32(bound or 0), None if acc is None else _ptr(acc), _ptr(out))
    return out


def emu_insert_absent(emu, table, pks, idx, accepted=None):
    t = np.array(table, np.uint32)
    ix = np.array(idx, np.uint32)
    inserted = np.zeros(max(len(ix), 1), np.uint8)
    acc = None if accepted is None else np.array(accepted, np.uint8)
    emu.emu_insert_absent(_ptr(t), ctypes.c_uint32(len(t)), _ptr(_blob(pks)), _ptr(ix), ctypes.c_size_t(len(ix)),
                          None if acc is None else _ptr(acc), _ptr(inserted))
    return t, inserted[:len(ix)].astype(bool)


def key_set(rng, n, dup_frac=0.3):
    """n keys of 32 bytes, about dup_frac of them repeating an earlier one."""
    distinct = [rng.bytes(32) for _ in range(n)]
    return [distinct[rng.integers(0, i)] if i and rng.random() < dup_frac else distinct[i] for i in range(n)]


CASES = [(seed, n, extra) for seed, (n, extra) in enumerate([(1, 0), (7, 0), (8, 9), (16, 0), (31, 2), (100, 7), (257, 16), (1000, 63)])]


# ---------------------------------------------------------------------------------------------------- tests
def test_capacity_is_the_smallest_power_of_two_of_at_least_16_and_twice_the_slots(emu):
    for n in list(range(0, 70)) + [1000, 4096, 4352, 10000]:
        assert emu.emu_capacity(n) == capacity(n), n


@pytest.mark.parametrize("bits", [4, 9, 20])
def test_lone_key_sits_at_its_hash(emu, bits):
    """A lone key sits at key_hash & mask, for masks of up to 20 bits: the hash the device probe uses is the one restated here."""
    rng = np.random.default_rng(bits)
    for _ in range(8):
        k = rng.bytes(32)
        table = emu_build(emu, [k], 1 << (bits - 1), [1])
        assert list(np.nonzero(table != NO_KEY)[0]) == [key_hash(k) & ((1 << bits) - 1)]


@pytest.mark.parametrize("seed,n,extra", CASES)
def test_build_matches_linear_probing(emu, seed, n, extra):
    """Every key slot in service, none, and random masks; the table sized for the slots plus spares, as a registration sizes it."""
    rng = np.random.default_rng(100 + seed)
    pks = key_set(rng, n)
    masks = [[1] * n, [0] * n] + [list(rng.random(n) < p) for p in (0.2, 0.5, 0.9)]
    for m in masks:
        got = emu_build(emu, pks, n + extra, m)
        assert got.tolist() == ref_build(pks, n + extra, m)
        # the first of equal key bytes wins: each in-service key's bytes reach the lowest in-service slot holding them
        first = [min(j for j in range(n) if m[j] and pks[j] == pks[i]) if m[i] else NO_KEY for i in range(n)]
        found = emu_find(emu, got, pks, pks, bound=n)
        assert [f for f, keep in zip(found.tolist(), m) if keep] == [f for f in first if f != NO_KEY]


@pytest.mark.parametrize("seed,n,extra", CASES)
def test_find_with_both_accept_rules(emu, seed, n, extra):
    """accept = idx < n_keys (the latency path's lookup) and accept = the slot is live (hs_committee_update), over keys in the table,
    keys whose slot is not accepted, keys out of service and keys that are absent."""
    rng = np.random.default_rng(200 + seed)
    pks = key_set(rng, n)
    in_service = list(rng.random(n) < 0.8)
    table = ref_build(pks, n + extra, in_service)
    assert emu_build(emu, pks, n + extra, in_service).tolist() == table
    queries = pks + [rng.bytes(32) for _ in range(max(4, n // 4))]
    for bound in sorted({0, 1, n // 2, n, n + extra}):
        got = emu_find(emu, table, pks, queries, bound=bound)
        want = [ref_find(table, pks, q, lambda s: s < bound) for q in queries]
        assert got.tolist() == want, bound
    for p in (0.0, 0.5, 1.0):
        live = list(rng.random(n) < p)
        got = emu_find(emu, table, pks, queries, accepted=live)
        want = [ref_find(table, pks, q, lambda s: live[s]) for q in queries]
        assert got.tolist() == want, p
    assert (emu_find(emu, table, pks, queries[n:], bound=n + extra) == NO_KEY).all()  # absent keys


@pytest.mark.parametrize("seed,n,extra", CASES)
def test_insert_absent_in_index_order_equals_build(emu, seed, n, extra):
    """Learning keys one call at a time (insert_absent of each new slot, in order) gives the table a rebuild over them gives, and
    reports exactly the first slot of each key as inserted."""
    rng = np.random.default_rng(300 + seed)
    pks = key_set(rng, n)
    table = [NO_KEY] * capacity(n + extra)
    cuts = sorted({0, n} | set(rng.integers(0, n + 1, 3).tolist()))
    for lo, hi in zip(cuts, cuts[1:]):
        table, inserted = emu_insert_absent(emu, table, pks, list(range(lo, hi)))
        assert inserted.tolist() == [pks.index(pks[i]) == i for i in range(lo, hi)]
    assert table.tolist() == ref_build(pks, n + extra, [1] * n)


@pytest.mark.parametrize("seed,n,extra", CASES)
def test_insert_absent_accepting_live_slots(emu, seed, n, extra):
    """hs_committee_update's step: a key whose only equal slot is not live is inserted again, and find then reaches it."""
    rng = np.random.default_rng(400 + seed)
    extra = max(extra, 4)
    pks = key_set(rng, n) + [rng.bytes(32) for _ in range(extra)]
    table = ref_build(pks, n + extra, [1] * n)                        # the published table
    live = [bool(rng.random() < 0.6) for _ in range(n)] + [True] * extra  # removals since, and the spare slots added
    held = {pks[j] for j in range(n) if live[j]}
    removed = list({pks[i]: i for i in range(n) if pks[i] not in held}.values())  # one slot per key no live slot holds
    for k in range(min(len(removed), extra // 2)):                    # a removed key added again into a spare slot
        pks[n + k] = pks[removed[k]]
    pks[n + extra - 1] = pks[n - 1]                                   # a published key added again
    new = list(range(n, n + extra))
    got, inserted = emu_insert_absent(emu, table, pks, new, accepted=live)
    ref = list(table)
    assert inserted.tolist() == [ref_insert_absent(ref, pks, i, lambda s: live[s]) for i in new] and got.tolist() == ref
    assert inserted.tolist()[:min(len(removed), extra // 2)] == [True] * min(len(removed), extra // 2)
    found = emu_find(emu, got, pks, [pks[i] for i in new], accepted=live)
    assert all(live[f] and pks[f] == pks[i] for f, i in zip(found.tolist(), new))


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_committee_update_gives_equal_keys_one_slot():
    """hs_committee_update looks each added key up in the published index plus the keys the call already added: a key added twice in one
    call takes one slot, also when the same call removed it; the published table then passes the audit against the node's map."""
    from hotstuff_b200 import Engine
    eng = Engine(0, base_window=12, key_window=8)  # small comb tables: the footprint stays small on a shared device
    try:
        seeds = np.frombuffer(np.random.default_rng(5).bytes(32 * 34), np.uint8).reshape(34, 32).copy()
        pks = eng.keygen_batch(seeds)
        assert eng.committee_register(pks[:32]).all()
        node = [bytes(k) for k in pks[:32]]
        idx = eng.committee_update(np.stack([pks[32], pks[32]]))                  # a new key twice: one spare slot
        assert list(idx) == [32, 32]
        node.append(bytes(pks[32]))
        idx = eng.committee_update(np.stack([pks[20], pks[20]]), remove=[5, 20])  # a removed key back twice: one slot, the lowest freed
        assert list(idx) == [5, 5]
        node[5], node[20] = bytes(pks[20]), None
        idx = eng.committee_update(np.stack([pks[33], pks[20], pks[33]]))         # a live key again, and a new one twice
        assert list(idx) == [20, 5, 20]
        node[20] = bytes(pks[33])
        assert eng.key_slots == len(node) == 33
        expect = np.stack([np.frombuffer(k, np.uint8) for k in node])
        failed, bits = eng.table_audit(expect)
        assert failed == 0 and not bits.any(), eng.last_error
    finally:
        eng.close()
