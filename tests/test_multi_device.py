"""Multi-device context (hs_multi_*, hotstuff_b200.MultiEngine): one process, several member contexts, host-pointer verify calls sharded
across them.  On one H100 the members are [0, 0]: two contexts on one GPU, with a 16-bit base window and 12-bit key windows so that their
tables fit beside each other.  Every output must equal the single-context call on the same device and the oracle, bit for bit, on both
sides of the sharding threshold; small calls must run on one member, round-robin, and sharded ones on every member."""
import ctypes
import os
import threading

import numpy as np
import pytest

from oracle_api import make_adversarial, make_workload, to_rec128
from test_groups_dev import K, expected, keys, make_burst  # noqa: F401 (keys is a fixture)

MIN = 4096  # HS_MULTI_MIN_SHARD
WIN = dict(base_window=16, key_window=12, key_cache=False)
SMALL = [1, 31, 64, 65, 2 * MIN - 1]
SHARDED = [2 * MIN, 2 * MIN + 1, 20000, 1 << 17]


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import build
    build.build_engine()


@pytest.fixture(scope="module")
def multi():
    _gpu()
    from hotstuff_b200 import MultiEngine
    m = MultiEngine([0, 0], **WIN)
    yield m
    m.close()


@pytest.fixture(scope="module")
def single():
    _gpu()
    from hotstuff_b200 import Engine
    e = Engine(0, **WIN)
    yield e
    e.close()


@pytest.fixture(scope="module")
def work(oracle):
    """2^17 records over 64 keys with 2 % corrupted, and 300 adversarial records spread through them; oracle verdicts in both modes."""
    w = make_workload(oracle, 1 << 17, n_keys=64, seed=77, corrupt_frac=0.02)
    recs = to_rec128(w)
    adv = make_adversarial(oracle, 300, seed=78)
    pos = np.random.default_rng(79).choice(recs.shape[0], adv.shape[0], replace=False)
    recs[pos] = adv
    return dict(recs=recs, pks=w["pks"], want=[oracle.verify_rec128(recs, mode=m) for m in (0, 1)])


def _launches(m):
    return [m.member(i).kernel_launches for i in range(len(m))]


def _moved(m, before):
    return [a - b for a, b in zip(_launches(m), before)]


def _clear(*engines):
    for e in engines:
        (e.register_committee if hasattr(e, "register_committee") else e.committee_register)(np.zeros((0, 32), np.uint8))


def _check_routing(moved, n):
    if n // 2 >= MIN:
        assert all(d > 0 for d in moved), moved
    else:
        assert sorted(d > 0 for d in moved) == [False, True], moved


# ---- rec128
@pytest.mark.gpu
@pytest.mark.parametrize("committee", [True, False])
@pytest.mark.parametrize("n", SMALL + SHARDED)
def test_rec128_parity_and_routing(multi, single, work, committee, n):
    recs = work["recs"][:n]
    if committee:
        assert multi.register_committee(work["pks"]).all() and single.committee_register(work["pks"]).all()
    try:
        for mode in (0, 1):
            before = _launches(multi)
            got = multi.verify_rec128(recs, mode)
            _check_routing(_moved(multi, before), n)
            assert (got == work["want"][mode][:n]).all(), np.flatnonzero(got != work["want"][mode][:n])[:8]
            assert (got == single.verify_rec128(recs, mode)).all()
    finally:
        _clear(multi, single)


@pytest.mark.gpu
def test_small_calls_alternate_members(multi, work):
    assert multi.register_committee(work["pks"]).all()
    try:
        seen = []
        for k in range(4):
            before = _launches(multi)
            assert (multi.verify_rec128(work["recs"][:8], 0) == work["want"][0][:8]).all()
            moved = _moved(multi, before)
            assert sorted(d > 0 for d in moved) == [False, True], moved
            assert max(moved) == 1  # up to 64 records with registered keys: the one-launch latency path
            seen.append(int(np.argmax(moved)))
        assert seen[0] != seen[1] and seen[1] != seen[2] and seen[2] != seen[3], seen
    finally:
        _clear(multi)


# ---- msgs
def _msgs(oracle, pks_all, n, seed):
    rng = np.random.default_rng(seed)
    msg_len = 100
    msgs = rng.integers(0, 256, (n, msg_len), dtype=np.uint8)
    seeds = np.random.default_rng(77).integers(0, 256, size=(64, 32), dtype=np.uint8)  # make_workload's keys (seed 77, 64 keys)
    kidx = rng.integers(0, 64, n).astype(np.uint32)
    dg = oracle.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * msg_len)
    sig = oracle.sign_batch(seeds, pks_all, kidx, dg.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    bad = rng.choice(n, max(1, n // 50), replace=False)
    sig[bad, 3] ^= 0x10
    recs = np.concatenate([sig, pks_all[kidx], dg], axis=1)
    return sig, msgs, msg_len, kidx, [oracle.verify_rec128(recs, mode=m) for m in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 65, 2 * MIN - 1, 2 * MIN, 20000])
def test_msgs_parity(multi, single, oracle, work, n):
    sig, msgs, msg_len, kidx, want = _msgs(oracle, work["pks"], n, n)
    pk = work["pks"][kidx]
    for committee in (False, True):
        if committee:
            assert multi.register_committee(work["pks"]).all() and single.committee_register(work["pks"]).all()
        try:
            for mode in (0, 1):
                forms = [dict(pk=pk)] + ([dict(validator_idx=kidx)] if committee else [])
                for form in forms:
                    before = _launches(multi)
                    got = multi.verify_msgs(sig, msgs.reshape(-1), msg_len, mode=mode, **form)
                    _check_routing(_moved(multi, before), n)
                    assert (got == want[mode]).all(), (mode, list(form), np.flatnonzero(got != want[mode])[:8])
                    assert (got == single.verify_msgs(sig, msgs.reshape(-1), msg_len, mode=mode, **form)).all()
        finally:
            _clear(multi, single)


# ---- groups
def _groups(e, b, indexed, modes, want_items):
    return e.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"] if modes else None,
                           pk=None if indexed else b["pk"], validator_idx=b["kidx"] if indexed else None, want_items=want_items)


def _check_groups(multi, single, oracle, keys, b, indexed):
    n = len(b["mi"])
    for modes in (True, False):
        want_g, want_i = expected(oracle, keys, b, indexed, modes)
        before = _launches(multi)
        g, items = _groups(multi, b, indexed, modes, True)
        _check_routing(_moved(multi, before), n)
        sg, si = _groups(single, b, indexed, modes, True)
        assert (items == si).all() and (g == sg).all(), (np.flatnonzero(items != si)[:8], np.flatnonzero(g != sg)[:8])
        assert (items == want_i).all() and (g == want_g).all()
        assert (_groups(multi, b, indexed, modes, False) == want_g).all()  # no item bitmap
    return want_g, want_i


@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["committee", "indexed", "none"])
@pytest.mark.parametrize("n", [1, 31, 64, 65, 2 * MIN - 1, 2 * MIN, 2 * MIN + 1, 20000])
def test_groups_parity(multi, single, oracle, keys, setup, n):
    """Mixed-mode Blocks, Timeout bursts and TCs, with records whose strict and batch-eq verdicts differ, against hs_verify_groups on one
    context and the oracle: key bytes with a registered committee, the committee-indexed form, key bytes without a committee."""
    b = make_burst(oracle, keys, np.random.default_rng(5000 + n + len(setup)), n)
    if setup != "none":
        assert multi.register_committee(keys[1][:K]).all() and single.committee_register(keys[1][:K]).all()
    try:
        want_g, _ = _check_groups(multi, single, oracle, keys, b, setup == "indexed")
        assert want_g[-1]  # the trailing group has no items
    finally:
        _clear(multi, single)


@pytest.mark.gpu
def test_groups_across_the_shard_boundary(multi, single, oracle, keys):
    """At n = 2 * MIN the boundary is item MIN.  Group A spans it with a rejected item left of it only, group B with one right of it only,
    group C spans it with nothing rejected, group D has no items.  The members' group words are ANDed on the host."""
    n = 2 * MIN
    b = make_burst(oracle, keys, np.random.default_rng(31337), n, corrupt=0.0)
    G = b["n_groups"]
    A, B, C, D = G, G + 1, G + 2, G + 3
    b["n_groups"] = G + 4
    b["gi"][MIN - 16:MIN + 16] = A
    b["gi"][MIN - 32:MIN - 16] = B
    b["gi"][MIN + 16:MIN + 32] = B
    b["gi"][MIN - 48:MIN - 32] = C
    b["gi"][MIN + 32:MIN + 48] = C
    items = expected(oracle, keys, b, False, True)[1] & expected(oracle, keys, b, False, False)[1]  # accepted in its mode and strict
    good = int(np.flatnonzero(items[:MIN - 200])[0])
    for i in np.flatnonzero((b["gi"] == C) & ~items):  # C must be accepted: give any rejected item of it an accepted item's record
        b["sig"][i], b["pk"][i], b["mi"][i], b["modes"][i] = b["sig"][good], b["pk"][good], b["mi"][good], b["modes"][good]
    b["sig"][MIN - 5, 40] ^= 1  # A: left of the boundary
    b["sig"][MIN + 20, 40] ^= 1  # B: right of it
    assert multi.register_committee(keys[1][:K]).all() and single.committee_register(keys[1][:K]).all()
    try:
        want_g, want_i = _check_groups(multi, single, oracle, keys, b, False)
        assert not want_i[MIN - 5] and not want_i[MIN + 20]
        assert not want_g[A] and not want_g[B] and want_g[D]
        assert want_g[C]
    finally:
        _clear(multi, single)


# ---- registration
@pytest.mark.gpu
def test_register_and_update_match_one_context(multi, single, oracle):
    rng = np.random.default_rng(99)
    seeds = rng.integers(0, 256, (300, 32), dtype=np.uint8)
    pks = oracle.keygen_batch(seeds)
    pks[[7, 150]] = np.frombuffer(bytes([2]) + bytes(31), np.uint8)  # y = 2 does not decompress
    try:
        valid = multi.register_committee(pks)
        assert (valid == single.committee_register(pks)).all() and not valid[7] and not valid[150] and valid.sum() == 298
        assert [multi.member(i).window_bits[0] for i in range(2)] == [12, 12]
        add_seeds = rng.integers(0, 256, (20, 32), dtype=np.uint8)
        add = oracle.keygen_batch(add_seeds)
        add = np.concatenate([add, pks[3:4], add[5:6]])  # an already registered key and a repeat
        idx = multi.update_committee(add, remove=np.array([1, 2, 9], np.uint32))
        assert (idx == single.committee_update(add, remove=np.array([1, 2, 9], np.uint32))).all()
        assert idx[20] == 3 and idx[21] == idx[5]
        # the committee-indexed form after the update: every live index, reused and added ones included, signs with its own key
        key_seed = {i: seeds[i] for i in range(300) if i not in (1, 2, 7, 9, 150)}
        key_seed.update({int(idx[j]): add_seeds[j] for j in range(20)})
        live = np.array(sorted(key_seed), np.uint32)
        vidx = live[rng.integers(0, live.size, 2 * MIN + 5)]
        kseeds = np.array([key_seed[int(i)] for i in live], np.uint8)
        kpks = oracle.keygen_batch(kseeds)
        kidx = np.searchsorted(live, vidx).astype(np.uint32)
        msgs = rng.integers(0, 256, (vidx.size, 32), dtype=np.uint8)
        dg = oracle.digest32_batch(msgs.reshape(-1), np.arange(vidx.size + 1, dtype=np.uint64) * 32)
        sig = oracle.sign_batch(kseeds, kpks, kidx, dg.reshape(-1), np.arange(vidx.size + 1, dtype=np.uint64) * 32)
        sig[::97, 5] ^= 4
        want = oracle.verify_rec128(np.concatenate([sig, kpks[kidx], dg], axis=1))
        got = multi.verify_msgs(sig, msgs.reshape(-1), 32, validator_idx=vidx)
        assert (got == want).all() and (got == single.verify_msgs(sig, msgs.reshape(-1), 32, validator_idx=vidx)).all()
        assert want.sum() > 0.9 * vidx.size
    finally:
        _clear(multi, single)


@pytest.mark.gpu
def test_failed_registration_leaves_no_committee(oracle):
    """Member tables of 2.35 GB each (544 slots of 12-bit tables) with 3.5 GB of device memory free: exactly one member's table
    allocation fails (HS_ERR_NOMEM, no GPU fault), and the member that succeeded is cleared again.  Then registration works."""
    _gpu()
    import torch
    from hotstuff_b200 import EngineError, MultiEngine
    m = MultiEngine([0, 0], **WIN)
    try:
        pks = oracle.keygen_batch(np.random.default_rng(5).integers(0, 256, (512, 32), dtype=np.uint8))
        table = 544 * 22 * 2048 * 96  # capk x comb_table_entries(12) x sizeof(ge_niels)
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        filler = torch.empty(max(0, free - table * 3 // 2), dtype=torch.uint8, device="cuda")
        try:
            with pytest.raises(EngineError, match=r"member [01] \(device 0\)"):
                m.register_committee(pks)
        finally:
            del filler
            torch.cuda.empty_cache()
        assert [m.member(i).window_bits[0] for i in range(2)] == [0, 0]
        assert m.register_committee(pks).all()
        assert [m.member(i).window_bits[0] for i in range(2)] == [12, 12]
    finally:
        m.close()


# ---- argument errors and lifecycle
def _threads():
    return len(os.listdir("/proc/self/task"))


@pytest.mark.gpu
def test_create_failures_and_destroy_leave_no_thread():
    _gpu()
    from hotstuff_b200 import EngineError, MultiEngine, _lib
    lib = _lib.load()
    MultiEngine([0, 0], **WIN).close()  # the CUDA runtime's own threads start with the first context
    t0 = _threads()
    h = ctypes.c_void_p(1)
    devs = (ctypes.c_int * 2)(0, 0)
    assert lib.hs_multi_create(ctypes.byref(h), devs, 0, 16) == 2 and not h
    with pytest.raises(EngineError):
        MultiEngine([0, 999], **WIN)
    assert _threads() == t0
    for n in (1, 2, 3):
        m = MultiEngine([0] * n, **WIN)
        assert _threads() == t0 + n - 1 and len(m) == n
        m.close()
        assert _threads() == t0


@pytest.mark.gpu
def test_argument_errors_write_nothing(multi, work):
    lib = multi.lib
    S = 0xA5A5A5A5
    for n in (40, 2 * MIN):
        recs = np.ascontiguousarray(work["recs"][:n])
        out = np.full((n + 31) // 32, S, np.uint32)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        assert lib.hs_multi_verify_rec128(multi.h, p(recs), n, 2, p(out)) == 2 and (out == S).all()
        assert "hs_multi_verify_rec128: bad argument" in multi.last_error
        sig = np.ascontiguousarray(recs[:, :64])
        msgs = np.ascontiguousarray(recs[:, 96:])
        assert lib.hs_multi_verify_msgs(multi.h, p(sig), None, None, p(msgs), 32, n, 0, p(out)) == 2 and (out == S).all()
        assert lib.hs_multi_verify_msgs(multi.h, p(sig), p(np.ascontiguousarray(recs[:, 64:96])), None, p(msgs), 0, n, 0, p(out)) == 2
        assert (out == S).all()
        pre = np.zeros(64, np.uint8)
        off = np.array([0, 32, 64], np.uint64)
        mi = np.zeros(n, np.uint32)
        gi = (np.arange(n) % 3).astype(np.uint32)
        mo = np.zeros(n, np.uint8)
        pk = np.ascontiguousarray(recs[:, 64:96])
        gout = np.full(1, S, np.uint32)
        for bad in ("msg", "group", "mode", "offsets"):
            mi2, gi2, mo2, off2 = mi.copy(), gi.copy(), mo.copy(), off.copy()
            if bad == "msg":
                mi2[-1] = 2
            elif bad == "group":
                gi2[-1] = 3
            elif bad == "mode":
                mo2[-1] = 2
            else:
                off2[1] = 65
            rc = lib.hs_multi_verify_groups(multi.h, p(pre), p(off2), 2, p(sig), p(pk), None, p(mi2), p(gi2), p(mo2), n, 3, p(out), p(gout))
            assert rc == 2 and (out == S).all() and (gout == S).all(), bad
            assert "hs_multi_verify_groups: " in multi.last_error


# ---- concurrency
@pytest.mark.gpu
def test_queue_on_a_member_beside_sharded_calls(multi, work):
    """A verify queue on member 0 keeps giving oracle-equal verdicts while another thread runs sharded calls through the multi-context."""
    assert multi.register_committee(work["pks"]).all()
    errors = []
    n = 2 * MIN + 100

    def sharded():
        try:
            for k in range(6):
                got = multi.verify_rec128(work["recs"][:n], k & 1)
                if not (got == work["want"][k & 1][:n]).all():
                    errors.append("sharded call %d" % k)
        except Exception as e:  # noqa: BLE001 (reported below)
            errors.append(repr(e))

    q = multi.member(0).queue()
    try:
        t = threading.Thread(target=sharded)
        t.start()
        tickets = []
        for k in range(60):
            lo = (k * 37) % 5000
            tickets.append((lo, k & 1, q.submit(work["recs"][lo:lo + 16], mode=k & 1)))
        for lo, mode, tk in tickets:
            assert tk is not None
            assert (q.wait(tk) == work["want"][mode][lo:lo + 16]).all(), lo
        t.join()
        assert not errors, errors
    finally:
        q.close()
        _clear(multi)


# ---- two GPUs
@pytest.mark.gpu
def test_parity_on_two_gpus(oracle, keys, work):
    import torch
    _gpu()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from hotstuff_b200 import Engine, MultiEngine
    m, e = MultiEngine([0, 1], **WIN), Engine(0, **WIN)
    try:
        for n in (65, 2 * MIN, 20000):
            for mode in (0, 1):
                before = _launches(m)
                assert (m.verify_rec128(work["recs"][:n], mode) == work["want"][mode][:n]).all()
                _check_routing(_moved(m, before), n)
        b = make_burst(oracle, keys, np.random.default_rng(2), 20000)
        assert m.register_committee(keys[1][:K]).all() and e.committee_register(keys[1][:K]).all()
        for indexed in (False, True):
            _check_groups(m, e, oracle, keys, b, indexed)
    finally:
        m.close()
        e.close()
