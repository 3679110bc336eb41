"""hs_explain_groups_dev (Engine.explain_groups_dev): the table-free re-check of hs_explain_rec128 for the rejected items of a
device-resident hs_verify_groups_dev pass, with a why byte per item and an engine-fault count, nothing copied to the host.

CPU: the new symbols agree across the header, the ctypes table, the Python constants, the C++ mirror and the Rust submodule; the ordered
selection under host emulation (tests/hostemu/explain_select_emu.cpp, the kernels' own index helpers) equals a plain Python selection on
random, all-zero and all-one bitmaps with ragged last words and caps of 1, 31, 32, 33 and above the count; the engine-fault rule equals
the Rust shim's.
GPU: masks of mixed Block / Timeout / TC passes with golden vectors, adversarial records and small-order keys equal hs_explain_rec128 on
the host-built records and the oracle's masks; a clean engine reports no fault; the cap takes the lowest-index rejected items; cleared
bits of valid items and a poked flag byte are reported as engine faults; deferred mode needs no host wait; the call leaves the queue,
the key cache and later verdicts alone and host-pointer calls do not wait for it; argument errors write nothing."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from oracle_api import make_adversarial
from test_binding_consistency import _strip_comments, header_functions
from test_explain import Expect
from test_groups_dev import K, _clear, _digests, _register, enqueue, keys, make_burst, to_device  # noqa: F401  (keys: a fixture)
from test_table_repair import POKE_FLAG, _engine, _poke, hooklib  # noqa: F401  (hooklib: the -DHS_TEST_HOOKS build, a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_EXAMINED, SMALL = 0x80, 8 | 16
NONE = 0xffffffff


def valid_in_mode(why, mode):
    """The Rust shim's engine-fault rule (explain_rejected): batch-eq allows only the small-order bits; every other mode byte is strict."""
    return (why & ~SMALL & 0xff) == 0 if mode == 1 else why == 0


# ---------------------------------------------------------------------------------------------------- CPU: bindings
def test_symbols_agree_across_the_bindings():
    from hotstuff_b200 import _lib, engine
    fns = header_functions()
    assert fns["hs_explain_groups_dev"] == ("int", ["hs_ctx*", "const void*", "const void*", "size_t", "const void*", "const void*", "const void*",
                                                    "const void*", "const void*", "size_t", "size_t", "void*", "void*", "void*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_WHY_NOT_EXAMINED 0x80u\b", hdr) and re.search(r"#define HS_EXPLAIN_DEV_OUT 4\b", hdr)
    c_void_p, c_size_t = ctypes.c_void_p, ctypes.c_size_t
    assert _lib.SIGNATURES["hs_explain_groups_dev"] == (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p,
                                                                       c_void_p, c_size_t, c_size_t, c_void_p, c_void_p, c_void_p])
    assert engine.WHY_NOT_EXAMINED == 0x80 and engine.EXPLAIN_DEV_OUT == 4 and callable(engine.Engine.explain_groups_dev)
    # C++ mirror: one call with every argument, in the header's order
    hpp = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.hpp")).read())
    call = re.search(r"hs_explain_groups_dev\((.*?)\)", hpp, flags=re.S).group(1)
    assert [a.strip() for a in call.split(",")] == ["ctx_", "d_preimages", "d_pre_off", "n_msgs", "d_sig", "d_pk", "d_msg_idx", "d_mode_or_null",
                                                    "d_item_bitmap", "n_items", "max_explain", "d_why", "d_out", "stream"]
    # Rust: its own submodule, extern block matching the header, constants matching, a failed call never read as success
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_explain_dev.rs"\]\s*pub mod explain_dev;', shim)
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_explain_dev.rs")).read())
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    rust_to_c = {"*mut HsCtx": "hs_ctx*", "*const c_void": "const void*", "*mut c_void": "void*", "usize": "size_t", "c_int": "int"}
    found = re.findall(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*->\s*([^;]+);", block, flags=re.S)
    assert [f[0] for f in found] == ["hs_explain_groups_dev"]
    name, params, ret = found[0]
    assert [rust_to_c[re.sub(r"\s+", " ", p.split(":", 1)[1].strip())] for p in params.split(",") if p.strip()] == fns[name][1]
    assert rust_to_c[ret.strip()] == "int"
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == {"hs_explain_groups_dev"}
    assert "pub const HS_WHY_NOT_EXAMINED: u8 = 0x80;" in src and "pub const HS_EXPLAIN_DEV_OUT: usize = 4;" in src
    assert "rc == HS_OK" in src and "pub unsafe fn explain_rejected_dev(ctx: *mut HsCtx, g: &DevGroups" in src


# ---------------------------------------------------------------------------------------------------- CPU: the selection
@pytest.fixture(scope="module")
def selemu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("selemu") / "libhs_selemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "explain_select_emu.cpp")])
    emu = ctypes.CDLL(lib)
    emu.emu_select.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
    emu.emu_valid_in_mode.restype = ctypes.c_uint32
    return emu


def _select(emu, words, n, cap):
    words = np.ascontiguousarray(words, np.uint32)
    lst = np.full(n + 1, 0xdeadbeef, np.uint32)
    out = np.zeros(2, np.uint32)
    emu.emu_select(words.ctypes.data, n, cap, lst.ctypes.data, out.ctypes.data)
    return out, lst


@pytest.mark.parametrize("n", [1, 31, 32, 33, 95, 8191, 8192, 8193, 8192 * 3 + 17, 70000])
def test_selection_matches_a_plain_reference(selemu, n):
    rng = np.random.default_rng(n)
    n_words = (n + 31) // 32
    for kind in ("random", "sparse", "zeros", "ones"):
        if kind == "random":
            words = rng.integers(0, 2**32, n_words, dtype=np.uint64).astype(np.uint32)
        elif kind == "sparse":  # about 1 % of the bits 0
            bits = rng.random(n_words * 32) >= 0.01
            words = np.packbits(bits, bitorder="little").view(np.uint32)
        else:
            words = np.full(n_words, 0 if kind == "zeros" else 0xffffffff, np.uint32)
        if n % 32 and kind != "zeros":  # the high bits past n are ignored, whatever they hold
            words[-1] |= np.uint32(0xffffffff << (n % 32) & 0xffffffff)
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:n]
        zero = np.flatnonzero(bits == 0)
        for cap in sorted({0, 1, 31, 32, 33, len(zero), len(zero) + 1, len(zero) + 40}):
            out, lst = _select(selemu, words, n, cap)
            want = zero if cap == 0 else zero[:cap]
            assert out[0] == len(zero) and out[1] == len(want), (kind, cap)
            assert (lst[:len(want)] == want).all(), (kind, cap)
            assert (lst[len(want):] == 0xdeadbeef).all(), (kind, cap)  # nothing past the selection is written


def test_fault_rule_matches_the_rust_shim(selemu):
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert "if modes[index] == HS_MODE_BATCH_EQ { why & !(HS_WHY_A_SMALL | HS_WHY_R_SMALL) == 0 } else { why == 0 }" in shim
    for why in range(256):
        for mode in (0, 1, 2, 7, 255):
            assert bool(selemu.emu_valid_in_mode(why, mode)) == valid_in_mode(why, mode), (why, mode)


# ---------------------------------------------------------------------------------------------------- GPU helpers
def with_records(b, sig, pk, msgs, where):
    """The pass b with items `where` replaced by the records (sig, pk) over preimages msgs (each its own new preimage)."""
    b = dict(b)
    pres = [b["pre"]] + [np.frombuffer(bytes(m), np.uint8) for m in msgs]
    lens = [len(m) for m in msgs]
    off = np.concatenate([b["off"], b["off"][-1] + np.cumsum(lens, dtype=np.uint64)]).astype(np.uint64)
    n_old = len(b["off"]) - 1
    b["pre"], b["off"] = np.concatenate(pres).astype(np.uint8), off
    b["sig"], b["pk"], b["mi"], b["kidx"] = b["sig"].copy(), b["pk"].copy(), b["mi"].copy(), b["kidx"].copy()
    b["sig"][where], b["pk"][where] = sig, pk
    b["mi"][where] = np.arange(n_old, n_old + len(where), dtype=np.uint32)
    b["kidx"][where] = K
    return b


def records(b):
    """The (n, 128) records the engine judges: sig, key bytes, Digest of the item's preimage."""
    n = len(b["mi"])
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = b["sig"], b["pk"], _digests(b["pre"], b["off"])[b["mi"]]
    return recs


def mixed_pass(oracle, keys, golden, n, seed):
    """make_burst's Blocks, Timeouts and TCs (corrupted items, small-order keys in both modes) with golden vectors and adversarial records
    in place of some items, each over its own message as a preimage."""
    rng = np.random.default_rng(seed)
    b = make_burst(oracle, keys, rng, n, corrupt=0.02)
    gv = golden["vectors"]
    adv = make_adversarial(oracle, max(1, min(n // 3, 400)), seed=seed)
    sig = [np.frombuffer(bytes.fromhex(v["sig"]), np.uint8) for v in gv] + [r[:64] for r in adv]
    pk = [np.frombuffer(bytes.fromhex(v["pk"]), np.uint8) for v in gv] + [r[64:96] for r in adv]
    msgs = [bytes.fromhex(v["msg"]) for v in gv] + [r[96:].tobytes() for r in adv]
    m = min(len(sig), max(1, n // 3))
    pick = rng.permutation(len(sig))[:m]
    where = np.sort(rng.choice(n, m, replace=False))
    sig, pk, msgs = [sig[k] for k in pick], [pk[k] for k in pick], [msgs[k] for k in pick]
    return with_records(b, np.stack(sig), np.stack(pk), msgs, where)


def explain(engine, b, d, ib, max_explain=0, modes=True):
    import torch
    n = len(b["mi"])
    why = torch.full((n,), 0x11, dtype=torch.uint8, device="cuda")
    out = torch.full((4,), 0x7777, dtype=torch.int32, device="cuda")
    engine.explain_groups_dev(d["pre"], d["off"], len(b["off"]) - 1, d["sig"], d["pk_bytes"], d["mi"], ib, n, why, out,
                              d_mode=d["mode"] if modes else None, max_explain=max_explain)
    return why, out


def dev(b):
    import torch
    d = to_device(b)
    d["pk_bytes"] = torch.from_numpy(np.ascontiguousarray(b["pk"])).cuda()
    return d


def _bools(t, n):
    return np.unpackbits(t.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def _u32(out):
    return out.cpu().numpy().view(np.uint32)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 32, 33, 2500, 70000])
def test_masks_match_host_explain_and_the_oracle(engine, oracle, keys, golden, n):
    """Every rejected item's mask equals hs_explain_rec128 on the host-built record and the oracle's expected mask, in both mode forms;
    every accepted item reads HS_WHY_NOT_EXAMINED; a clean engine reports no fault."""
    import torch
    b = mixed_pass(oracle, keys, golden, n, seed=7 * n + 1)
    recs = records(b)
    want = Expect(oracle).recs(recs)
    _register(engine, keys)
    try:
        d = dev(b)
        for modes in (True, False):
            mode_bytes = b["modes"] if modes else np.zeros(n, np.uint8)
            ib = enqueue(engine, b, dict(d, mode=d["mode"] if modes else None))[0]
            why, out = explain(engine, b, d, ib, modes=modes)
            torch.cuda.synchronize()
            items, why, out = _bools(ib, n), why.cpu().numpy(), _u32(out)
            ok = np.array([valid_in_mode(int(w), int(m)) for w, m in zip(want, mode_bytes)], bool)
            assert (items == ok).all()  # the pass itself agrees with the oracle: this engine is clean
            rej = np.flatnonzero(~items)
            assert (why[items] == NOT_EXAMINED).all()
            assert (why[rej] == want[rej]).all(), rej[why[rej] != want[rej]][:8]
            if rej.size:
                assert (why[rej] == engine.explain(recs[rej])).all()
            assert list(out) == [rej.size, rej.size, 0, NONE]
        if n >= 2500:
            assert ((want & SMALL) != 0).any() and (want & 0x27).any() and (b["modes"] == 1).any() and (b["modes"] == 0).any()
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_cap_takes_the_lowest_index_rejected_items(engine, oracle, keys, golden):
    import torch
    b = mixed_pass(oracle, keys, golden, 2500, seed=99)
    want = Expect(oracle).recs(records(b))
    _register(engine, keys)
    try:
        d = dev(b)
        ib = enqueue(engine, b, d)[0]
        torch.cuda.synchronize()
        rej = np.flatnonzero(~_bools(ib, 2500))
        assert rej.size > 64
        for cap in (1, 31, 32, 33, 64, rej.size, rej.size + 10):
            why, out = explain(engine, b, d, ib, max_explain=cap)
            torch.cuda.synchronize()
            why, out = why.cpu().numpy(), _u32(out)
            pick = rej[:cap]
            assert list(out) == [rej.size, pick.size, 0, NONE], cap
            assert (why[pick] == want[pick]).all(), cap
            rest = np.setdiff1d(np.arange(2500), pick)
            assert (why[rest] == NOT_EXAMINED).all(), cap
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_cleared_bits_of_valid_items_are_engine_faults(engine, oracle, keys, golden):
    """A bitmap with the bits of valid items cleared counts exactly those items as faults and reports the lowest; a batch-eq-only item
    (small-order R or A, equation holds) is a fault under mode byte 1 only, not when the mode array is NULL (all strict)."""
    import torch
    b = mixed_pass(oracle, keys, golden, 2500, seed=5)
    want = Expect(oracle).recs(records(b))
    _register(engine, keys)
    try:
        d = dev(b)
        ib = enqueue(engine, b, d)[0]
        torch.cuda.synchronize()
        items = _bools(ib, 2500)
        eq_only = np.flatnonzero(items & (b["modes"] == 1) & (want != 0))  # accepted under batch-eq, rejected strict
        plain = np.flatnonzero(items & (want == 0))
        assert eq_only.size and plain.size > 40
        rng = np.random.default_rng(3)
        flip = np.sort(np.concatenate([rng.choice(plain, 40, replace=False), eq_only[:3]]))
        bits = items.copy()
        bits[flip] = False
        words = torch.from_numpy(np.packbits(np.pad(bits, (0, (-2500) % 32)), bitorder="little").view(np.int32).copy()).cuda()
        why, out = explain(engine, b, d, words)
        torch.cuda.synchronize()
        out, why = _u32(out), why.cpu().numpy()
        rej = np.flatnonzero(~bits)
        assert list(out) == [rej.size, rej.size, flip.size, flip.min()]
        assert (why[flip] == want[flip]).all()
        why, out = explain(engine, b, d, words, modes=False)  # every item strict: the batch-eq-only items are rightly rejected
        torch.cuda.synchronize()
        strict_faults = np.setdiff1d(flip, eq_only)
        assert list(_u32(out)) == [rej.size, rej.size, strict_faults.size, strict_faults.min()]
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_a_poked_flag_byte_is_reported_as_an_engine_fault(hooklib, oracle, keys):
    """On the hook build: a live slot's flag byte poked so its key reads as not decompressing; hs_verify_groups_dev then rejects that
    key's honest items, and the explanation reports each of them (and nothing else) as an engine fault."""
    import torch
    e = _engine(hooklib, base_window=16)
    try:
        b = make_burst(oracle, keys, np.random.default_rng(11), 600, corrupt=0.0)
        e.committee_register(keys[1][:K])
        d = dev(b)
        ib = enqueue(e, b, d)[0]
        torch.cuda.synchronize()
        clean = _bools(ib, 600)
        slot = int(b["kidx"][np.flatnonzero(clean & (b["kidx"] < K))[0]])
        _poke(e, POKE_FLAG, slot, 0, 0x01)
        ib = enqueue(e, b, d)[0]
        why, out = explain(e, b, d, ib)
        torch.cuda.synchronize()
        items, out, why = _bools(ib, 600), _u32(out), why.cpu().numpy()
        faults = np.flatnonzero(clean & ~items)
        assert faults.size and (b["kidx"][faults] == slot).all()
        assert list(out) == [(~items).sum(), (~items).sum(), faults.size, faults.min()]
        assert all(valid_in_mode(int(why[i]), int(b["modes"][i])) for i in faults)
    finally:
        e.close()


@pytest.mark.gpu
def test_deferred_pass_then_explanation_without_a_host_wait(engine, oracle, keys, golden):
    import torch
    b = mixed_pass(oracle, keys, golden, 3000, seed=21)
    _register(engine, keys)
    try:
        d = dev(b)
        ib = enqueue(engine, b, d)[0]
        why0, out0 = explain(engine, b, d, ib)
        torch.cuda.synchronize()
        engine.set_deferred(True)
        try:
            for _ in range(3):  # the item words come from the tail stream; the explanation follows on the caller's stream
                ib2 = enqueue(engine, b, d)[0]
                why, out = explain(engine, b, d, ib2)
            torch.cuda.synchronize()
        finally:
            engine.set_deferred(False)
        assert (why.cpu() == why0.cpu()).all() and (out.cpu() == out0.cpu()).all() and _u32(out0)[0] > 0
    finally:
        _clear(engine)


@pytest.mark.gpu
def test_isolation_and_no_wait_for_host_calls(engine, oracle, keys, golden):
    """The queue's stats, hs_cached_keys and the verdicts of a following pass are unchanged by explanations, and a host-pointer verify
    issued while a large explanation runs on another stream returns before it ends."""
    import torch
    b = mixed_pass(oracle, keys, golden, 2500, seed=31)
    recs = records(b)
    _register(engine, keys)
    q = engine.queue()
    try:
        d = dev(b)
        ib = enqueue(engine, b, d)[0]
        torch.cuda.synchronize()
        before_items = _bools(ib, 2500)
        st, cached = q.stats(), engine.cached_keys
        launches = engine.kernel_launches
        explain(engine, b, d, ib)
        torch.cuda.synchronize()
        assert engine.kernel_launches == launches + 4
        assert q.stats() == st and engine.cached_keys == cached
        assert (_bools(enqueue(engine, b, d)[0], 2500) == before_items).all()
        # a large all-rejected explanation on a side stream: 2^18 items, every bit 0
        n = 1 << 18
        big = dict(b)
        rep = -(-n // 2500)
        big = dict(pre=b["pre"], off=b["off"], sig=np.tile(b["sig"], (rep, 1))[:n], pk=np.tile(b["pk"], (rep, 1))[:n],
                   mi=np.tile(b["mi"], rep)[:n], kidx=np.tile(b["kidx"], rep)[:n], gi=np.zeros(n, np.uint32), modes=np.tile(b["modes"], rep)[:n],
                   n_groups=1)
        dbig = dev(big)
        zeros = torch.zeros(n // 32, dtype=torch.int32, device="cuda")
        want_small = engine.verify_rec128(recs[:48])
        side = torch.cuda.Stream()
        explain(engine, big, dbig, zeros, max_explain=64)  # grows the scratch for the big call (may synchronise) before the timing
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            why, out = explain(engine, big, dbig, zeros)
            done = torch.cuda.Event()
            done.record(side)
        got = engine.verify_rec128(recs[:48])
        still_running = not done.query()
        torch.cuda.synchronize()
        assert (got == want_small).all()
        assert still_running, "the host-pointer call waited for the explanation"
        assert list(_u32(out))[:2] == [n, n]
    finally:
        q.close()
        _clear(engine)


@pytest.mark.gpu
def test_argument_errors_write_nothing(engine, oracle, keys, golden):
    import torch
    from hotstuff_b200 import EngineError
    b = mixed_pass(oracle, keys, golden, 100, seed=41)
    d = dev(b)
    ib = torch.zeros(4, dtype=torch.int32, device="cuda")
    why = torch.full((100,), 0x11, dtype=torch.uint8, device="cuda")
    out = torch.full((4,), 0x7777, dtype=torch.int32, device="cuda")
    m = len(b["off"]) - 1
    args = [d["pre"], d["off"], m, d["sig"], d["pk_bytes"], d["mi"], ib, 100, why, out]
    launches = engine.kernel_launches
    for k in (0, 1, 3, 4, 5, 6, 8, 9):
        bad = list(args)
        bad[k] = None
        with pytest.raises(EngineError):
            engine.explain_groups_dev(*bad)
    bad = list(args)
    bad[2] = 0
    with pytest.raises(EngineError):
        engine.explain_groups_dev(*bad)
    bad = list(args)
    bad[7] = 0  # no items: HS_OK, nothing written, nothing launched
    engine.explain_groups_dev(*bad)
    torch.cuda.synchronize()
    assert engine.kernel_launches == launches
    assert (why.cpu() == 0x11).all() and (out.cpu() == 0x7777).all()
    engine.explain_groups_dev(*args)  # the context is still usable
    torch.cuda.synchronize()
    assert _u32(out)[0] == 100 and (why.cpu() != 0x11).all()
