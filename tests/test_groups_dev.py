"""hs_verify_groups_dev (Engine.verify_groups_dev) + hs_qc_and_dev: hs_verify_groups with every array in device memory.  Item bits (each
item in its own verdict mode, judged by k_verify_finish_modes) and group bits must equal hs_verify_groups on the same arrays bit for bit,
and the oracle, for Blocks with and without a TC, view-change bursts of Timeouts sharing one high_qc, and TCs, with about 1 % of records
corrupted in the signature, the key or the preimage.  Also: deferred mode over a stream of passes, the peer route at world 1, a sharded
burst over two GPUs (hotstuff_b200.sharding.verify_groups_sharded), host-checkable argument errors, and on the CPU the shard arithmetic
of the sharded pass over gloo."""
import ctypes
import hashlib
import os
import socket
import sys

import numpy as np
import pytest

from oracle_api import L_ORDER

HERE = os.path.dirname(os.path.abspath(__file__))
K, FOREIGN = 256, 8  # committee keys, then keys that are never registered


@pytest.fixture(scope="module")
def keys(oracle):
    rng = np.random.default_rng(4242)
    seeds = rng.integers(0, 256, size=(K + FOREIGN, 32), dtype=np.uint8)
    return seeds, oracle.keygen_batch(seeds)


def _digests(pre, off):
    return np.array([np.frombuffer(hashlib.sha512(pre[int(off[j]):int(off[j + 1])]).digest()[:32], np.uint8) for j in range(len(off) - 1)]).reshape(-1, 32)


def make_burst(oracle, keys, rng, n_items, corrupt=0.01, foreign=False):
    """Exactly n_items items in groups: Blocks (author strict over a Block preimage, QC votes batch-eq over 40 bytes, with or without TC
    votes strict over 16 bytes each), view-change bursts (Timeouts, each its author strict over 16 bytes plus the SAME high_qc's votes
    batch-eq) and TCs (votes strict over 16 bytes each), some groups with no items.  `corrupt` of the items get a flipped bit in the
    signature, the key or their preimage (after signing).  foreign: one item is signed by a key outside the committee."""
    seeds, pks = keys
    pres, mi, modes, gi, dup = [], [], [], [], []
    g = 0

    def pre(b):
        pres.append(b)
        return len(pres) - 1

    def add(m, mode, same_as=-1):
        mi.append(m)
        modes.append(mode)
        gi.append(g)
        dup.append(same_as)
        return len(mi) - 1

    while len(mi) < n_items:
        kind = int(rng.integers(4))
        if kind < 2:  # Block, with a TC when kind == 1
            add(pre(rng.bytes(int(rng.integers(60, 400)))), 0)
            q = pre(rng.bytes(40))
            for _ in range(int(rng.integers(2, 40))):
                add(q, 1)
            for _ in range(int(rng.integers(2, 20)) if kind == 1 else 0):
                add(pre(rng.bytes(16)), 0)
            g += 1
        elif kind == 2:  # Timeouts carrying one high_qc: its votes are the same records in every Timeout
            q = pre(rng.bytes(40))
            first = None
            for _ in range(int(rng.integers(2, 8))):
                add(pre(rng.bytes(16)), 0)
                votes = [add(q, 1, -1 if first is None else first[k]) for k in range(len(first) if first else int(rng.integers(2, 30)))]
                first = first or votes
                g += 1
        else:  # TC
            for _ in range(int(rng.integers(2, 30))):
                add(pre(rng.bytes(16)), 0)
            g += 1
        if rng.random() < 0.2:
            g += 1  # a group with no items
    n = n_items
    mi, gi = np.array(mi[:n], np.uint32), np.array(gi[:n], np.uint32)
    modes, dup = np.array(modes[:n], np.uint8), np.array(dup[:n], np.int64)
    off = np.zeros(len(pres) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in pres])
    pre_b = np.frombuffer(b"".join(pres), np.uint8).copy()
    kidx = rng.integers(0, K, n).astype(np.uint32)
    for i in np.flatnonzero(dup >= 0):
        kidx[i] = kidx[dup[i]]  # the same vote in every Timeout of the burst (Ed25519 signatures are deterministic)
    if foreign:  # an item that no other item copies
        lone = np.setdiff1d(np.flatnonzero(dup < 0), dup)
        kidx[lone[int(rng.integers(len(lone)))]] = K + int(rng.integers(FOREIGN))
    dig = _digests(pre_b, off)
    sig = oracle.sign_batch(seeds, pks, kidx, dig[mi].reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32)
    pk = pks[kidx].copy()
    for i in np.flatnonzero(rng.random(n) < corrupt):
        what = int(rng.integers(3))
        if what == 0:
            sig[i, int(rng.integers(64))] ^= np.uint8(1 << int(rng.integers(8)))
        elif what == 1:
            pk[i, int(rng.integers(32))] ^= np.uint8(1 << int(rng.integers(8)))
        elif off[mi[i] + 1] > off[mi[i]]:
            pre_b[int(rng.integers(off[mi[i]], off[mi[i] + 1]))] ^= np.uint8(1 << int(rng.integers(8)))
    small_order_items(oracle, keys, rng, sig, pk, kidx, modes, _digests(pre_b, off)[mi])
    return dict(pre=pre_b, off=off, sig=sig, pk=pk, kidx=kidx, mi=mi, gi=gi, modes=modes, n_groups=g + 1)  # the last group has no items


IDENTITY = (1).to_bytes(32, "little")              # y = 1: the neutral element
ORDER2 = (2**255 - 19 - 1).to_bytes(32, "little")  # y = -1: the point of order 2


def small_order_items(oracle, keys, rng, sig, pk, kidx, modes, msgs, frac=0.03):
    """Replaces about `frac` of the committee-signed items of each mode (at least one) with records over their own message on which
    strict and batch-eq may disagree.  The first in each mode is a registered key with R = the identity and S = k * a: the cofactorless
    equation holds, so batch-eq accepts it and strict rejects it for its small-order R, whether the key is given by bytes or by index.
    The others are R = the identity and S = 0 under a small-order key (the identity: the equation holds; the point of order 2: it
    holds when k is even)."""
    seeds, pks = keys
    for mode in (0, 1):
        idx = np.flatnonzero((modes == mode) & (kidx < K))
        if idx.size == 0:
            continue
        for j, i in enumerate(rng.choice(idx, max(1, int(frac * idx.size)), replace=False)):
            m = msgs[i].tobytes()
            if j == 0 or rng.random() < 0.3:
                h = hashlib.sha512(seeds[kidx[i]].tobytes()).digest()
                a = int.from_bytes(bytes([h[0] & 248]) + h[1:31] + bytes([(h[31] & 127) | 64]), "little")
                k = oracle.sc_reduce64(hashlib.sha512(IDENTITY + pks[kidx[i]].tobytes() + m).digest())
                sig[i] = np.frombuffer(IDENTITY + (k * a % L_ORDER).to_bytes(32, "little"), np.uint8)
                pk[i] = pks[kidx[i]]
            else:
                sig[i] = np.frombuffer(IDENTITY + bytes(32), np.uint8)
                pk[i] = np.frombuffer(IDENTITY if rng.random() < 0.5 else ORDER2, np.uint8)


def both_modes(oracle, keys, b, indexed=False):
    """The oracle's strict and batch-eq verdicts of every item."""
    n = len(b["mi"])
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = b["sig"], keys[1][b["kidx"]] if indexed else b["pk"], _digests(b["pre"], b["off"])[b["mi"]]
    return oracle.verify_rec128(recs, mode=0), oracle.verify_rec128(recs, mode=1)


def assert_modes_matter(oracle, keys, b, indexed=False, modes=None):
    """Every mode byte present among the committee-signed items has an item whose strict and batch-eq verdicts differ, so a finish
    kernel that ignored the byte, or read it the wrong way round, would get that item wrong."""
    modes = b["modes"] if modes is None else modes
    strict, eq = both_modes(oracle, keys, b, indexed)
    for m in np.unique(modes[b["kidx"] < K]):
        assert ((strict != eq) & (modes == m)).any(), "no item in mode byte %d tells strict from batch-eq" % m


def expected(oracle, keys, b, indexed=False, modes=True):
    """The oracle's item verdicts over the (possibly corrupted) preimages, each in its mode, and the group ANDs."""
    strict, eq = both_modes(oracle, keys, b, indexed)
    items = np.where(b["modes"] == 1, eq, strict) if modes else strict  # any byte but HS_MODE_BATCH_EQ is strict
    groups = np.ones(b["n_groups"], bool)
    np.logical_and.at(groups, b["gi"], items)
    return groups, items


def _bools(t, n):
    return np.unpackbits(t.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def to_device(b, indexed=False, modes=True):
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return dict(pre=t(b["pre"] if b["pre"].size else np.zeros(1, np.uint8)), off=t(b["off"].view(np.int64)), sig=t(b["sig"]),
                pk=None if indexed else t(b["pk"]), vidx=t(b["kidx"].view(np.int32)) if indexed else None, mi=t(b["mi"].view(np.int32)),
                gi=t(b["gi"].view(np.int32)), mode=t(b["modes"]) if modes else None)


def enqueue(engine, b, d):
    """One hs_verify_groups_dev pass and its group AND on torch's stream; returns the (item, group) bitmap tensors."""
    import torch
    n, G = len(b["mi"]), b["n_groups"]
    ib = torch.zeros(max(1, (n + 31) // 32), dtype=torch.int32, device="cuda")
    gb = torch.zeros(max(1, (G + 31) // 32), dtype=torch.int32, device="cuda")
    engine.verify_groups_dev(d["pre"], d["off"], len(b["off"]) - 1, d["sig"], d["mi"], ib, n, d_mode=d["mode"], d_pk=d["pk"], d_vidx=d["vidx"])
    engine.qc_and_dev(ib, d["gi"], n, G, gb)
    return ib, gb


def run_dev(engine, b, indexed=False, modes=True):
    import torch
    ib, gb = enqueue(engine, b, to_device(b, indexed, modes))
    torch.cuda.synchronize()
    return _bools(gb, b["n_groups"]), _bools(ib, len(b["mi"]))


def run_host(engine, b, indexed=False, modes=True):
    return engine.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"] if modes else None,
                                pk=None if indexed else b["pk"], validator_idx=b["kidx"] if indexed else None, want_items=True)


def _register(engine, keys):
    assert engine.committee_register(keys[1][:K]).all()  # in order: committee index = key index


def _clear(engine):
    engine.committee_register(np.zeros((0, 32), np.uint8))


# ---- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["committee", "foreign", "indexed", "none"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 2500])
def test_parity_with_verify_groups_and_the_oracle(engine, oracle, keys, setup, n):
    """Item and group bits equal hs_verify_groups and the oracle, with modes and with mode == NULL: key bytes with a registered committee,
    with one foreign key in the pass, the committee-indexed form, and key bytes without a committee (twice: the key cache learns)."""
    rng = np.random.default_rng(1000 * n + len(setup))
    b = make_burst(oracle, keys, rng, n, foreign=setup == "foreign")
    indexed = setup == "indexed"
    assert_modes_matter(oracle, keys, b, indexed)
    if setup == "none":
        _clear(engine)
    else:
        _register(engine, keys)
    try:
        for modes in (True, False):
            want_g, want_i = expected(oracle, keys, b, indexed, modes)
            for _ in range(2 if setup == "none" else 1):
                g, items = run_dev(engine, b, indexed, modes)
                hg, hi = run_host(engine, b, indexed, modes)
                assert (items == hi).all() and (g == hg).all(), (np.flatnonzero(items != hi)[:8], np.flatnonzero(g != hg)[:8])
                assert (items == want_i).all() and (g == want_g).all()
        assert g[-1]  # the trailing group has no items
        if n >= 2500:
            assert (~want_i).sum() > 0 and want_i.sum() > 0 and (b["modes"] == 1).any() and (b["modes"] == 0).any()
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_mode_bytes_other_than_batch_eq_are_strict(engine, oracle, keys):
    """The strict items' mode bytes replaced by 2, 255, 0 and 7 (the host form rejects bytes above 1, the device form cannot see them):
    every such item is judged strict, so the bits equal hs_verify_groups with those bytes set to 0, and the oracle."""
    rng = np.random.default_rng(255)
    b = make_burst(oracle, keys, rng, 1500)
    odd = b["modes"].copy()
    strict_items = np.flatnonzero(odd != 1)
    odd[strict_items] = np.array([2, 255, 0, 7], np.uint8)[np.arange(strict_items.size) % 4]
    strict, eq = both_modes(oracle, keys, b)
    special = np.flatnonzero(strict != eq)
    odd[special[b["modes"][special] != 1]] = 255  # every strict item that tells the modes apart gets an odd byte
    assert ((strict != eq) & (odd > 1)).any() and ((strict != eq) & (odd == 1)).any()
    _register(engine, keys)
    try:
        want_g, want_i = expected(oracle, keys, b)
        hg, hi = run_host(engine, b)
        g, items = run_dev(engine, dict(b, modes=odd))
        assert (items == hi).all() and (g == hg).all() and (items == want_i).all() and (g == want_g).all()
        assert (items[special] == np.where(odd[special] == 1, eq[special], strict[special])).all()
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_deferred_stream_of_passes(engine, oracle, keys):
    """24 passes of different sizes on one caller stream in deferred mode, closed by ONE hs_results_wait: every pass's item and group
    bits equal hs_verify_groups (run before the stream) and the oracle."""
    import torch
    rng = np.random.default_rng(77)
    _register(engine, keys)
    sizes = [int(x) for x in rng.permutation([1, 5, 31, 32, 33, 64, 100, 257, 700, 1500, 3000, 40] * 2)]
    bursts = [make_burst(oracle, keys, rng, n, foreign=k % 5 == 0) for k, n in enumerate(sizes)]
    for b in bursts:
        assert_modes_matter(oracle, keys, b)
    want = [expected(oracle, keys, b) for b in bursts]
    host = [run_host(engine, b) for b in bursts]
    devs = [to_device(b) for b in bursts]
    torch.cuda.synchronize()
    engine.set_deferred(True)
    try:
        outs = [enqueue(engine, b, d) for b, d in zip(bursts, devs)]
        engine.results_wait()
        torch.cuda.synchronize()
    finally:
        engine.set_deferred(False)
        _clear(engine)
    for b, (ib, gb), (wg, wi), (hg, hi) in zip(bursts, outs, want, host):
        g, items = _bools(gb, b["n_groups"]), _bools(ib, len(b["mi"]))
        assert (items == hi).all() and (g == hg).all() and (items == wi).all() and (g == wg).all(), len(b["mi"])


@pytest.mark.gpu
def test_peer_route_at_world_one(oracle, keys):
    """hs_peer_setup(rank 0, world 1) and hs_peer_next before each epoch: hs_peer_bitmap() holds the pass's item words and the group AND
    over it is right; an empty pass with the route armed still publishes its epoch flag."""
    import torch
    from hotstuff_b200 import Engine
    e = Engine(0, base_window=12)
    try:
        _register(e, keys)
        rng = np.random.default_rng(31)
        bursts = [make_burst(oracle, keys, rng, n) for n in (900, 33, 1, 2000, 64)]
        total = max((len(b["mi"]) + 31) // 32 for b in bursts)
        h = (ctypes.c_uint8 * 64)()
        e._check(e.lib.hs_peer_setup(e.h, 0, 1, total, h), "hs_peer_setup")

        def view(words, base=None):
            class _Arr:
                __cuda_array_interface__ = {"shape": (words,), "typestr": "<i4", "data": (int(base or e.lib.hs_peer_bitmap(e.h)), False), "version": 3}
            return torch.as_tensor(_Arr(), device="cuda")

        for epoch, b in enumerate(bursts, start=1):
            d = to_device(b)
            e._check(e.lib.hs_peer_next(e.h, 0, epoch), "hs_peer_next")
            local = torch.zeros(total, dtype=torch.int32, device="cuda")
            e.verify_groups_dev(d["pre"], d["off"], len(b["off"]) - 1, d["sig"], d["mi"], local, len(b["mi"]), d_mode=d["mode"], d_pk=d["pk"])
            full = view(total)
            gb = torch.zeros((b["n_groups"] + 31) // 32, dtype=torch.int32, device="cuda")
            e.qc_and_dev(full, d["gi"], len(b["mi"]), b["n_groups"], gb)
            torch.cuda.synchronize()
            wg, wi = expected(oracle, keys, b)
            assert (_bools(full, len(b["mi"])) == wi).all() and (_bools(gb, b["n_groups"]) == wg).all(), epoch
            assert not local.any()  # an armed pass stores into the peers' buffers, not the local bitmap
        # an empty pass with the route armed: the epoch flag (buffer word 2 * total + rank) still advances
        epoch = len(bursts) + 1
        e._check(e.lib.hs_peer_next(e.h, 0, epoch), "hs_peer_next")
        e.verify_groups_dev(d["pre"], d["off"], 0, d["sig"], d["mi"], local, 0)
        torch.cuda.synchronize()
        base = e.lib.hs_peer_bitmap(e.h) - (epoch & 1) * total * 4
        assert int(view(2 * total + 1, base)[2 * total]) == epoch
        assert not e.lib.hs_peer_timed_out(e.h)
    finally:
        e.close()


@pytest.mark.gpu
def test_argument_errors_leave_the_context_usable(engine, oracle, keys):
    """Host-checkable bad arguments return HS_ERR_ARG with a message; a correct pass follows on the same context."""
    import torch
    rng = np.random.default_rng(3)
    b = make_burst(oracle, keys, rng, 40)
    d = to_device(b)
    bm = torch.zeros(2, dtype=torch.int32, device="cuda")
    s = engine._stream()
    p = lambda t: t.data_ptr()
    lib, h, n, m = engine.lib, engine.h, len(b["mi"]), len(b["off"]) - 1
    good = [h, p(d["pre"]), p(d["off"]), m, p(d["sig"]), p(d["pk"]), None, p(d["mi"]), p(d["mode"]), n, p(bm), s]
    _clear(engine)
    for k in (1, 2, 4, 7, 10):  # preimages, offsets, signatures, message indices, item bitmap
        args = list(good)
        args[k] = None
        assert lib.hs_verify_groups_dev(*args) == 2 and b"hs_verify_groups_dev" in lib.hs_last_error(h)
    args = list(good)
    args[5] = None  # neither keys nor indices
    assert lib.hs_verify_groups_dev(*args) == 2
    args[3] = 0
    args[5] = good[5]
    assert lib.hs_verify_groups_dev(*args) == 2  # items without preimages
    args = list(good)
    args[5], args[6] = None, p(torch.from_numpy(b["kidx"].view(np.int32)).cuda())
    assert lib.hs_verify_groups_dev(*args) == 2 and b"committee" in lib.hs_last_error(h)  # indexed without a committee
    assert lib.hs_verify_groups_dev(None, *good[1:]) == 2
    assert lib.hs_verify_groups_dev(h, None, None, 0, None, None, None, None, None, 0, None, s) == 0  # nothing to do
    g, items = run_dev(engine, b)
    wg, wi = expected(oracle, keys, b)
    assert (g == wg).all() and (items == wi).all()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _burst_for_ranks(n):
    from oracle_api import Oracle
    o = Oracle()
    rng = np.random.default_rng(555)
    seeds = rng.integers(0, 256, size=(K + FOREIGN, 32), dtype=np.uint8)
    keys = (seeds, o.keygen_batch(seeds))
    return o, keys, make_burst(o, keys, rng, n, foreign=True)


def _gpu_worker(rank, world, port, n, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch
    import torch.distributed as dist
    from hotstuff_b200 import Engine
    from hotstuff_b200.sharding import PeerAllGather, verify_groups_sharded
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    o, keys, b = _burst_for_ranks(n)
    e = Engine(rank, base_window=12)
    _register(e, keys)
    single_g, single_i = run_host(e, b)  # the single-GPU result on this rank
    want_g, want_i = expected(o, keys, b)
    d = to_device(b)
    ok = bool((single_g == want_g).all() and (single_i == want_i).all())
    peer = PeerAllGather(e, n, rank, world)
    for use_peer in (True, False):
        for deferred in (True, False):
            e.set_deferred(deferred)
            gb = torch.zeros((b["n_groups"] + 31) // 32, dtype=torch.int32, device="cuda")
            full = verify_groups_sharded(e, d["pre"], d["off"], d["sig"], d["mi"], d["gi"], b["n_groups"], gb, rank, world, d_mode=d["mode"],
                                         d_pk=d["pk"], peer=peer if use_peer else None)
            if deferred:
                e.results_wait()
            torch.cuda.synchronize()
            ok = ok and bool((_bools(gb, b["n_groups"]) == single_g).all() and (_bools(full, n) == single_i).all())
            dist.barrier()
    e.set_deferred(False)
    ok = ok and not e.lib.hs_peer_timed_out(e.h)
    np.save(os.path.join(out_dir, "ok_%d.npy" % rank), np.array([ok]))
    dist.barrier()
    dist.destroy_process_group()
    e.close()


@pytest.mark.gpu
def test_sharded_mixed_burst_two_gpus(tmp_path):
    """A mixed burst sharded over two GPUs, through the fused peer stores and through the ncclAllGather fallback, with and without
    deferred mode: every rank's group and item bits equal the single-GPU hs_verify_groups result."""
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.spawn(_gpu_worker, args=(2, _free_port(), 3001, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        assert np.load(os.path.join(str(tmp_path), "ok_%d.npy" % r))[0], "rank %d: sharded group bits differ from the single-GPU pass" % r


# ---- CPU: the shard arithmetic of verify_groups_sharded over gloo, with a stand-in engine
class _ShardRecorder:
    """Engine stand-in on CPU tensors: verify_groups_dev writes item_ok's bits for the items it is handed (found from where the shard's
    views start in the full arrays) and records the range; qc_and_dev ANDs over the bitmap it is given with the group indices it is given."""

    def __init__(self, full, item_ok):
        self.full, self.item_ok, self.calls, self.and_calls, self.events = full, item_ok, [], [], []

    def verify_groups_dev(self, d_pre, d_off, n_msgs, d_sig, d_msg_idx, d_item_bitmap, n_items, d_mode=None, d_pk=None, d_vidx=None):
        import torch
        lo = (d_msg_idx.data_ptr() - self.full["mi"].data_ptr()) // 4 if n_items else None
        if n_items:
            assert (d_sig.data_ptr() - self.full["sig"].data_ptr()) // 64 == lo and (d_mode.data_ptr() - self.full["mode"].data_ptr()) == lo
            assert (d_pk.data_ptr() - self.full["pk"].data_ptr()) // 32 == lo and d_vidx is None
        assert d_pre is self.full["pre"] and d_off is self.full["off"] and n_msgs == self.full["off"].numel() - 1  # preimages whole
        bits = np.concatenate([self.item_ok[lo:lo + n_items] if n_items else np.zeros(0, bool), np.zeros((-n_items) % 32, bool)])
        words = np.frombuffer(np.packbits(bits, bitorder="little").tobytes(), dtype=np.int32)
        d_item_bitmap[: words.size] = torch.from_numpy(words.copy())
        self.calls.append((lo, n_items, d_item_bitmap.numel()))
        self.events.append("verify")

    def results_wait(self):
        self.events.append("wait")

    def qc_and_dev(self, d_vote_bitmap, d_qc_idx, n_votes, n_qc, d_qc_bitmap):
        import torch
        items = _bools(d_vote_bitmap, n_votes)
        g = np.ones(n_qc, bool)
        np.logical_and.at(g, d_qc_idx.numpy()[:n_votes], items)
        words = np.frombuffer(np.packbits(np.concatenate([g, np.zeros((-n_qc) % 32, bool)]), bitorder="little").tobytes(), dtype=np.int32)
        d_qc_bitmap[:] = torch.from_numpy(words.copy())
        self.and_calls.append((d_qc_idx is self.full["gi"], n_votes, n_qc))
        self.events.append("and")


def _gloo_worker(rank, world, port, n, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch
    import torch.distributed as dist
    from hotstuff_b200.sharding import shard_range, verify_groups_sharded
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(n)  # identical on every rank
    n_groups = max(1, n // 7) + 2
    gi = rng.integers(0, n_groups - 2, n).astype(np.int32)  # the last two groups have no items
    item_ok = rng.random(n) > 0.05
    full = dict(pre=torch.zeros(64, dtype=torch.uint8), off=torch.arange(0, 65, 16, dtype=torch.int64), sig=torch.zeros((n, 64), dtype=torch.uint8),
                pk=torch.zeros((n, 32), dtype=torch.uint8), mi=torch.zeros(n, dtype=torch.int32), gi=torch.from_numpy(gi), mode=torch.zeros(n, dtype=torch.uint8))
    e = _ShardRecorder(full, item_ok)
    gb = torch.zeros((n_groups + 31) // 32, dtype=torch.int32)
    got_items = _bools(verify_groups_sharded(e, full["pre"], full["off"], full["sig"], full["mi"], full["gi"], n_groups, gb, rank, world, d_mode=full["mode"],
                                             d_pk=full["pk"]), n)
    lo, hi, per = shard_range(n, rank, world)
    want_g = np.ones(n_groups, bool)
    np.logical_and.at(want_g, gi, item_ok)
    (call_lo, call_n, local_words), = e.calls
    ok = [per % 32 == 0, call_n == hi - lo, call_lo in (lo, None), local_words == max(1, per // 32),  # a contiguous range of whole words
          lo == min(n, rank * per),                                                                   # rank r's words start at word r * per / 32
          e.and_calls == [(True, n, n_groups)],                                                      # the whole group_idx goes to the AND
          e.events == ["verify", "wait", "and", "wait"],  # the fallback: tail stream -> collective, and the AND before the gathered buffer is reused
          bool((got_items == item_ok).all()), bool((_bools(gb, n_groups) == want_g).all()), bool(_bools(gb, n_groups)[-2:].all())]
    np.save(os.path.join(out_dir, "ok_%d.npy" % rank), np.array(ok))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n", [1, 33, 64, 1000])
def test_sharded_groups_arithmetic_gloo_world2(tmp_path, n):
    import torch.multiprocessing as mp
    mp.spawn(_gloo_worker, args=(2, _free_port(), n, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        ok = np.load(os.path.join(str(tmp_path), "ok_%d.npy" % r))
        assert ok.all(), "rank %d: checks %s failed" % (r, np.flatnonzero(~ok).tolist())


def test_bindings_match_the_header():
    """The header, the ctypes table, the Python method and the Rust submodule's extern block agree on hs_verify_groups_dev, and the
    submodule also declares and calls hs_qc_and_dev, the group AND (CPU)."""
    import re
    from test_binding_consistency import _strip_comments, header_functions
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import Engine
    root = os.path.dirname(HERE)
    want = ["hs_ctx*", "const void*", "const void*", "size_t", "const void*", "const void*", "const void*", "const void*", "const void*", "size_t",
            "void*", "void*"]
    fns = header_functions()
    assert fns["hs_verify_groups_dev"] == ("int", want)
    _, args = _lib.SIGNATURES["hs_verify_groups_dev"]
    assert [a is ctypes.c_size_t for a in args] == [t == "size_t" for t in want]
    assert callable(Engine.verify_groups_dev)
    shim = open(os.path.join(root, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_groups_dev.rs"\]\s*pub mod groups_dev;', shim)
    src = _strip_comments(open(os.path.join(root, "rust", "crypto_gpu_groups_dev.rs")).read())
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    rust_to_c = {"*mut HsCtx": "hs_ctx*", "*const c_void": "const void*", "*mut c_void": "void*", "usize": "size_t", "c_int": "int"}
    seen = set()
    for name, params, ret in re.findall(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*->\s*([^;]+);", block, flags=re.S):
        assert [rust_to_c[re.sub(r"\s+", " ", p.split(":", 1)[1].strip())] for p in params.split(",") if p.strip()] == fns[name][1], name
        assert rust_to_c[ret.strip()] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_verify_groups_dev", "hs_qc_and_dev"}
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    assert src.count("rc == HS_OK") == 2  # a failed call is an error, never an accept
