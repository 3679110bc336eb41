"""hs_committee_stage / hs_committee_commit / hs_committee_discard: a committee change prepared off the verify path and switched in with a
short commit.

GPU: stage(A, R) + commit leaves a context exactly as update(A) + update(remove=R) leaves another (indices, slots, audits, verdicts on
every path); nothing changes for verification before the commit; requests in flight across the commit complete with the oracle's
verdicts; registrations and updates invalidate a stage; a stage of any size costs the same launches, and so do an update's build and a
repair's rebuild; a vote burst beside a 256-key stage on a 4,096-key committee; a multi-device context stages and commits."""
import ctypes
import threading

import numpy as np
import pytest

from test_table_repair import POKE_TABLE, _engine, _entry_off, hooklib  # noqa: F401  (hooklib: the -DHS_TEST_HOOKS build, a fixture)

pytestmark = pytest.mark.gpu
HS_ERR_ARG, HS_ERR_NOMEM = 2, 3


def _keys(oracle, n, seed):
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    return seeds, oracle.keygen_batch(seeds)


def _bad_keys(oracle, n, seed):
    """n key encodings that do not decompress."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        k = np.frombuffer(rng.bytes(32), np.uint8).copy()
        k[31] &= 0x7f
        if not oracle.decompress_ok(k.tobytes()):
            out.append(k)
    return np.array(out, np.uint8)


def _sign(oracle, seeds, pks, ki, seed, corrupt=0.15, with_preimages=False):
    """Records by keys ki over the Digests of random 40-byte preimages, a share of them with a flipped signature bit."""
    rng = np.random.default_rng(seed)
    n = len(ki)
    pre = np.frombuffer(rng.bytes(40 * n), np.uint8).copy()
    dig = np.asarray(oracle.digest32_batch(pre, np.arange(n + 1, dtype=np.uint64) * 40), np.uint8).reshape(n, 32)
    sig = oracle.sign_batch(seeds, pks, np.asarray(ki, np.uint32), dig.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    recs = np.concatenate([sig, pks[ki], dig], axis=1)
    for i in np.nonzero(rng.random(n) < corrupt)[0]:
        recs[i, rng.integers(0, 64)] ^= 1 << rng.integers(0, 8)
    return (recs, pre) if with_preimages else recs


def _live_bits(live):
    w = np.zeros((len(live) + 31) // 32, np.uint32)
    for i, v in enumerate(live):
        if v:
            w[i // 32] |= np.uint32(1 << (i % 32))
    return w


class Node:
    """The node-side index -> key map: registration order, then every change's added indices and removals."""

    def __init__(self, pks):
        self.keys = [bytes(k) for k in pks]

    def apply(self, add, idx, remove=()):
        """stage(add, remove) + commit, or update(add) then update(remove=remove)."""
        for k, i in zip(add, idx):
            while i >= len(self.keys):
                self.keys.append(None)
            self.keys[i] = bytes(k)
        for i in remove:
            self.keys[i] = None

    def update(self, add, idx, remove=()):
        """One hs_committee_update(add, remove): its removals come first."""
        for i in remove:
            self.keys[i] = None
        self.apply(add, idx)

    def expect(self):
        exp = np.array([np.frombuffer(k, np.uint8) if k else np.zeros(32, np.uint8) for k in self.keys], np.uint8)
        return exp, _live_bits([k is not None for k in self.keys])


def _audit_clean(eng, node):
    exp, lv = node.expect()
    assert eng.key_slots == len(node.keys)
    failed, _ = eng.table_audit(exp, lv)
    assert failed == 0, eng.last_error


def _by_index(oracle, node, recs, vidx, mode=0):
    """The oracle's verdicts of committee-indexed records: the slot's key when it is in service, else reject."""
    want = np.zeros(len(recs), bool)
    for i, s in enumerate(vidx):
        k = node.keys[s] if s < len(node.keys) else None
        if k is not None:
            r = recs[i].copy()
            r[64:96] = np.frombuffer(k, np.uint8)
            want[i] = oracle.verify_rec128(r[None], mode=mode)[0]
    return want


def _every_path(eng, oracle, node, recs, pre, vidx):
    """Verdicts on every path equal the oracle's: key bytes in both modes (and through the latency path), committee indices, the
    queue's small and bulk kernels, hs_verify_groups and the self-test."""
    for mode in (0, 1):
        assert np.array_equal(eng.verify_rec128(recs, mode=mode), oracle.verify_rec128(recs, mode=mode))
    want = oracle.verify_rec128(recs)
    assert np.array_equal(eng.verify_rec128(recs[:48]), want[:48])
    got = eng.verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(recs), dtype=np.uint32))
    assert np.array_equal(got, _by_index(oracle, node, recs, vidx))
    q = eng.queue()
    try:
        small = [q.wait(q.submit(recs[i:i + 1]))[0] for i in range(min(len(recs), 64))]
        assert np.array_equal(np.array(small, bool), want[:len(small)])
        # at least 1,002 records whose keys are all in service: k_verify_bulk
        live = {k for k in node.keys if k is not None}
        inside = np.array([bytes(r[64:96]) in live for r in recs])
        grp = np.resize(recs[inside], (1024, 128))
        assert np.array_equal(q.wait(q.submit_group(grp)), np.resize(want[inside], 1024))
        st = q.stats()
        assert st["small_launches"] > 0 and st["bulk_launches"] > 0, st
    finally:
        q.close()
    # hs_verify_groups over the records' 40-byte preimages, by key bytes and by committee index, mixed modes
    n = len(recs)
    off = np.arange(n + 1, dtype=np.uint64) * 40
    modes = (np.arange(n) % 2).astype(np.uint8)
    gi = (np.arange(n) // 4).astype(np.uint32)
    ng = int(gi[-1]) + 1
    grecs = recs
    want_items = np.array([oracle.verify_rec128(grecs[i:i + 1], mode=int(modes[i]))[0] for i in range(n)])
    _, items = eng.verify_groups(pre, off, grecs[:, :64], np.arange(n, dtype=np.uint32), gi, ng, mode=modes, pk=grecs[:, 64:96], want_items=True)
    assert np.array_equal(items, want_items)
    want_idx = np.array([_by_index(oracle, node, grecs[i:i + 1], vidx[i:i + 1], mode=int(modes[i]))[0] for i in range(n)])
    _, items = eng.verify_groups(pre, off, grecs[:, :64], np.arange(n, dtype=np.uint32), gi, ng, mode=modes, validator_idx=vidx, want_items=True)
    assert np.array_equal(items, want_idx)
    assert eng.self_test() == 0, eng.last_error


def _committee(oracle, n, n_bad, seed):
    seeds, pks = _keys(oracle, n, seed)
    bad = _bad_keys(oracle, n_bad, seed + 1)
    pks[[17, 131][:n_bad]] = bad
    return seeds, pks


def test_stage_and_commit_equal_two_updates(oracle):
    """stage(A, R) + commit on one context, update(A) + update(remove=R) on another: the same indices, slots, clean audits against the
    same map, and the oracle's verdicts on every path, with records naming added, removed and reused indices."""
    from hotstuff_b200 import Engine
    seeds, pks = _committee(oracle, 300, 2, 500)
    nseeds, npks = _keys(oracle, 6, 501)
    bad = _bad_keys(oracle, 1, 502)
    e1, e2 = Engine(0, key_window=12), Engine(0, key_window=12)
    try:
        node = Node(pks)
        for e in (e1, e2):
            e.committee_register(pks)
            e.committee_update(remove=[20, 21])  # two free slots below the spares
        node.apply([], [], [20, 21])
        R = np.array([7, 9, 40, 41], np.uint32)
        # a registered key, a new key twice, a key whose slot is in R, a key that does not decompress, then new keys into the spares
        A = np.concatenate([pks[5:6], npks[0:1], npks[0:1], pks[7:8], bad, npks[1:6]])
        idx1 = e1.committee_stage(A, R)
        assert e1.key_slots == 300
        e1.committee_commit()
        idx2 = e2.committee_update(A)
        e2.committee_update(remove=R)
        assert np.array_equal(idx1, idx2)
        assert idx1[0] == 5 and idx1[1] == idx1[2] == 20 and idx1[3] == 7 and idx1[4] == 21 and list(idx1[5:]) == [300, 301, 302, 303, 304]
        node.apply(A, idx1, R)
        assert e1.key_slots == e2.key_slots == 305
        _audit_clean(e1, node)
        _audit_clean(e2, node)
        # records: added keys, removed keys, reused slots, old keys; committee indices name added, removed and reused slots
        all_seeds = np.concatenate([seeds, nseeds])
        all_pks = np.concatenate([pks, npks])
        ki = np.array(list(range(300, 306)) * 8 + [7, 9, 40, 41, 5, 20, 21, 17, 131, 0, 1, 2] * 6, np.int64)
        recs, pre = _sign(oracle, all_seeds, all_pks, ki, 503, with_preimages=True)
        new_slot = [idx1[1]] + list(idx1[5:])  # npks[0] sits in slot 20, npks[1:] in the spares
        vidx = np.array([new_slot[k - 300] if k >= 300 else k for k in ki], np.uint32)
        vidx[-6:] = 21  # the added key that does not decompress
        for e in (e1, e2):
            _every_path(e, oracle, node, recs, pre, vidx)
    finally:
        e1.close()
        e2.close()


def test_nothing_changes_before_the_commit(oracle):
    """Between stage and commit: the same verdicts, queue path counters and clean audit with the old map as before the stage; staged
    indices reject on the committee-indexed form; the commit then puts them in service."""
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 64, 510)
    nseeds, npks = _keys(oracle, 4, 511)
    e = Engine(0, key_window=12)
    try:
        e.committee_register(pks)
        node = Node(pks)
        all_seeds, all_pks = np.concatenate([seeds, nseeds]), np.concatenate([pks, npks])
        ki = np.array([64, 65, 66, 67, 0, 1, 2, 3] * 8)
        recs = _sign(oracle, all_seeds, all_pks, ki, 512, corrupt=0.0)

        def observe():
            v = [e.verify_rec128(recs, mode=m) for m in (0, 1)]
            q = e.queue()
            try:
                for i in range(len(recs)):
                    q.wait(q.submit(recs[i:i + 1]))
                st = q.stats()
            finally:
                q.close()
            return v, st

        before = observe()
        assert before[1]["slow_requests"] == 32  # the new keys' requests take the slow path
        idx = e.committee_stage(npks, [0, 1])
        assert list(idx) == [64, 65, 66, 67] and e.key_slots == 64
        after = observe()
        assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])) and before[1] == after[1]
        _audit_clean(e, node)
        sig, dig = recs[:, :64], recs[:, 96:]
        vidx = ki.astype(np.uint32)  # the staged indices are the spares 64..67
        got = e.verify_committee(vidx, sig, dig, msg_idx=np.arange(len(recs), dtype=np.uint32))
        assert not got[ki >= 64].any() and got[ki < 64].all()  # staged indices reject; removed validators 0 and 1 still verify
        e.committee_commit()
        node.apply(npks, idx, [0, 1])
        _audit_clean(e, node)
        got = e.verify_committee(vidx, sig, dig, msg_idx=np.arange(len(recs), dtype=np.uint32))
        assert np.array_equal(got, (ki >= 2))
    finally:
        e.close()


def test_requests_in_flight_across_the_commit(oracle):
    """Queue requests in flight during the commit complete with the oracle's verdicts; afterwards the added keys take the device path and
    removed indices reject."""
    from hotstuff_b200 import Engine
    seeds, pks = _keys(oracle, 24, 520)
    nseeds, npks = _keys(oracle, 4, 521)
    e = Engine(0, key_window=12)
    try:
        e.committee_register(pks)
        ki = np.arange(600) % 24
        recs = _sign(oracle, seeds, pks, ki, 522, corrupt=0.05)
        want = oracle.verify_rec128(recs)
        new_recs = _sign(oracle, nseeds, npks, np.arange(4), 523, corrupt=0.0)
        idx = e.committee_stage(npks, np.arange(4, dtype=np.uint32))
        with e.queue() as q:
            tickets = [(q.submit(recs[i:i + 3]), i) for i in range(0, 600, 3)]
            e.committee_commit()
            for t, i in tickets:
                assert (q.wait(t) == want[i:i + 3]).all()
            l0 = e.kernel_launches
            after = [q.submit(new_recs[i:i + 1]) for i in range(4)]
            assert all(q.wait(t).all() for t in after)
            assert e.kernel_launches - l0 <= 4  # device path: no generic-pass launches
        node = Node(pks)
        node.apply(npks, idx, range(4))
        vidx = np.arange(8, dtype=np.uint32)
        byidx = _sign(oracle, seeds, pks, np.arange(8), 524, corrupt=0.0)
        got = e.verify_committee(vidx, byidx[:, :64], byidx[:, 96:], msg_idx=np.arange(8, dtype=np.uint32))
        assert np.array_equal(got, _by_index(oracle, node, byidx, vidx))
        assert not got[:4].any() and got[4:].all()
    finally:
        e.close()


def test_invalidation_and_errors(oracle):
    from hotstuff_b200 import Engine, EngineError
    seeds, pks = _keys(oracle, 40, 530)
    _, npks = _keys(oracle, 80, 531)
    e = Engine(0, key_window=12)
    lib = e.lib
    try:
        # no committee
        with pytest.raises(EngineError):
            e.committee_stage(npks[:1])
        e.committee_register(pks)
        node = Node(pks)
        # an update between stage and commit: the commit refuses and changes nothing
        e.committee_stage(npks[:2], [3])
        idx = e.committee_update(npks[2:3], [4])
        node.update(npks[2:3], idx, [4])
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        _audit_clean(e, node)
        # a registration between stage and commit
        e.committee_stage(npks[:2])
        e.committee_register(pks)
        node = Node(pks)
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        _audit_clean(e, node)
        # a second stage is refused; discard frees the slots for the next stage
        first = e.committee_stage(npks[:3], [0])
        with pytest.raises(EngineError):
            e.committee_stage(npks[3:4])
        e.committee_discard()
        e.committee_discard()  # nothing staged: a no-op
        assert np.array_equal(e.committee_stage(npks[:3], [0]), first)
        e.committee_discard()
        _audit_clean(e, node)
        # HS_ERR_NOMEM leaves nothing staged: 40 keys, 16 spares
        out = np.full(17, 0xAAAAAAAA, np.uint32)
        add = np.ascontiguousarray(npks[:17])
        assert lib.hs_committee_stage(e.h, add.ctypes.data_as(ctypes.c_void_p), 17, None, 0, out.ctypes.data_as(ctypes.c_void_p)) == HS_ERR_NOMEM
        assert (out == 0xAAAAAAAA).all()
        assert lib.hs_committee_commit(e.h) == HS_ERR_ARG
        assert list(e.committee_stage(npks[:16])) == list(range(40, 56))
        e.committee_discard()
        # argument errors write nothing
        rem = np.array([56], np.uint32)  # past the slots in use once the additions are in
        out = np.full(16, 0xAAAAAAAA, np.uint32)
        add = np.ascontiguousarray(npks[:16])
        assert lib.hs_committee_stage(e.h, add.ctypes.data_as(ctypes.c_void_p), 16, rem.ctypes.data_as(ctypes.c_void_p), 1,
                                      out.ctypes.data_as(ctypes.c_void_p)) == HS_ERR_ARG
        assert lib.hs_committee_stage(e.h, None, 1, None, 0, out.ctypes.data_as(ctypes.c_void_p)) == HS_ERR_ARG
        assert lib.hs_committee_stage(e.h, add.ctypes.data_as(ctypes.c_void_p), 1, None, 0, None) == HS_ERR_ARG
        assert lib.hs_committee_stage(None, None, 0, None, 0, None) == HS_ERR_ARG
        assert lib.hs_committee_commit(None) == HS_ERR_ARG and lib.hs_committee_discard(None) == HS_ERR_ARG
        assert (out == 0xAAAAAAAA).all()
        # the last slot a stage's additions reach may be removed by it
        idx = e.committee_stage(npks[:16], [55])
        e.committee_commit()
        node.apply(npks[:16], idx, [55])
        _audit_clean(e, node)
    finally:
        e.close()


def test_an_update_racing_a_stage_ends_with_a_clean_audit(oracle):
    from hotstuff_b200 import Engine, EngineError
    seeds, pks = _keys(oracle, 400, 540)
    _, extra = _keys(oracle, 200, 541)  # 400 keys leave 25 spares: each stage takes 5
    e = Engine(0, key_window=12)
    try:
        e.committee_register(pks)
        node = Node(pks)
        outcomes = set()
        for it in range(4):
            add = extra[40 * it:40 * it + 5]
            res = {}

            def stage():
                try:
                    res["idx"] = e.committee_stage(add)
                except EngineError as err:
                    res["e"] = str(err)

            th = threading.Thread(target=stage)
            th.start()
            threading.Event().wait(0.002 * it)
            up = extra[40 * it + 30:40 * it + 31]
            idx = e.committee_update(up, [it])
            th.join()
            node.update(up, idx, [it])
            if "idx" in res:
                if e.lib.hs_committee_commit(e.h) == 0:  # staged after the update
                    node.apply(add, res["idx"])
                    outcomes.add("committed")
                else:  # staged before it: the update discarded it
                    outcomes.add("discarded")
            else:
                assert "during the stage" in res["e"], res["e"]
                outcomes.add("changed")
            _audit_clean(e, node)
        assert outcomes
    finally:
        e.close()


def test_launches_do_not_grow_with_the_slot_count(oracle, hooklib):
    """A stage costs one build and one proof launch for any K, an update's additions one build launch, and (hook build) a repair of K
    poked slots two audits plus one build and one proof."""
    from hotstuff_b200 import Engine
    _, pks = _keys(oracle, 64, 550)
    _, npks = _keys(oracle, 48, 551)
    e = Engine(0, key_window=12)
    try:
        e.committee_register(pks)
        e.committee_update(remove=np.arange(40, dtype=np.uint32))  # 40 free slots and 16 spares
        for K in (1, 7, 32):
            l0 = e.kernel_launches
            e.committee_stage(npks[:K])
            assert e.kernel_launches - l0 == 2, K
            e.committee_discard()
        for K, lo in ((1, 0), (7, 1), (32, 8)):
            l0 = e.kernel_launches
            e.committee_update(npks[lo:lo + K])
            assert e.kernel_launches - l0 == 1, K
    finally:
        e.close()
    h = _engine(hooklib, key_window=12)
    try:
        h.committee_register(pks)
        W = h.window_bits[0]
        for K in (1, 9):
            for s in range(10, 10 + K):
                assert hooklib.hs_test_poke(h.h, POKE_TABLE, s, _entry_off(W, 1, 3), 0x10) == 0
            l0 = h.kernel_launches
            found, failed, _ = h.table_repair(pks)
            assert failed == 0 and found, h.last_error
            assert h.kernel_launches - l0 == 2 * 3 + 2, K  # each audit: slots, tables, base table
    finally:
        h.close()


def test_votes_beside_a_256_key_stage(oracle):
    """A 667-vote queue burst from 16 threads while 256 keys are staged on a 4,096-key committee at the default window: every vote gets
    the oracle's verdict, and the stage commits to a clean audit."""
    from hotstuff_b200 import Engine
    e = Engine(0)
    try:
        rng = np.random.default_rng(560)
        seeds = np.frombuffer(rng.bytes(32 * 4096 + 32 * 256), np.uint8).reshape(-1, 32).copy()
        allpks = e.keygen_batch(seeds)
        pks, npks = allpks[:4096], allpks[4096:]
        e.committee_register(pks)
        node = Node(pks)
        rem = np.arange(1000, 1256, dtype=np.uint32)
        ki = rng.choice(4096, 667, replace=False)
        dig = np.frombuffer(rng.bytes(32), np.uint8)
        sig = e.sign_digests(seeds[:4096], pks, np.tile(dig, (667, 1)), key_idx=ki.astype(np.uint32))
        recs = np.concatenate([sig, pks[ki], np.tile(dig, (667, 1))], axis=1)
        for i in rng.choice(667, 40, replace=False):
            recs[i, rng.integers(0, 64)] ^= 1
        want = oracle.verify_rec128(recs)
        res = {}
        th = threading.Thread(target=lambda: res.setdefault("idx", e.committee_stage(npks, rem)))
        got = np.zeros(667, bool)
        with e.queue() as q:
            th.start()

            def worker(t):
                for i in range(t, 667, 16):
                    got[i] = q.wait(q.submit(recs[i:i + 1]))[0]

            ws = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
            for w in ws:
                w.start()
            for w in ws:
                w.join()
            th.join()
        assert np.array_equal(got, want)
        e.committee_commit()
        node.apply(npks, res["idx"], rem)
        _audit_clean(e, node)
    finally:
        e.close()


def test_multi_engine_stages_and_commits(oracle):
    from hotstuff_b200 import Engine, MultiEngine
    seeds, pks = _keys(oracle, 48, 570)
    nseeds, npks = _keys(oracle, 7, 571)
    m = MultiEngine([0, 0], key_window=12)
    single = Engine(0, key_window=12)
    try:
        m.register_committee(pks)
        single.committee_register(pks)
        R = np.array([1, 2, 9], np.uint32)
        idx = m.stage_committee(npks[:6], R)
        assert np.array_equal(idx, single.committee_stage(npks[:6], R))
        m.commit_committee()
        single.committee_commit()
        node = Node(pks)
        node.apply(npks[:6], idx, R)
        all_seeds, all_pks = np.concatenate([seeds, nseeds]), np.concatenate([pks, npks])
        ki = np.array(list(range(48, 54)) * 4 + [1, 2, 9, 0, 3], np.int64)
        recs = _sign(oracle, all_seeds, all_pks, ki, 572)
        vidx = np.array([idx[k - 48] if k >= 48 else k for k in ki], np.uint32)
        want = _by_index(oracle, node, recs, vidx)
        for i in range(len(m)):
            got = m.member(i).verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(recs), dtype=np.uint32))
            assert np.array_equal(got, want), i
            _audit_clean(m.member(i), node)
        # a discard on every member, then the same stage again
        again = m.stage_committee(npks[6:7])
        m.discard_committee()
        assert np.array_equal(m.stage_committee(npks[6:7]), again)
        m.discard_committee()
    finally:
        single.close()
        m.close()
