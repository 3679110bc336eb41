"""hs_table_audit: the audit of the live key tables.

CPU (host emulation, tests/hostemu/table_audit_emu.cpp): the per-entry checks k_table_audit runs, over tables built by comb_build_block, report every kind of corruption at
exactly the first bad (window, entry); the C++ and Rust wrappers exist and the Rust one switches the GPU off on a finding.
GPU: registered committees, committee updates and learned key-cache tables pass, with and without the caller's map; findings through
the expectation name the right slots; the audit is read-only and leaves the verify queue's verdicts and counters alone."""
import ctypes
import os
import re
import subprocess
import threading
import time

import numpy as np
import pytest

from oracle_api import P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = 96  # bytes of one affine Niels entry: ypx | ymx | xy2d


# ---------------------------------------------------------------------------------------------------- host emulation
def _valid_keys(hostemu, n, seed):
    rng = np.random.default_rng(seed)
    out, x, y = [], ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
    while len(out) < n:
        k = rng.bytes(32)
        if hostemu.emu_decompress(k, x, y):
            out.append(k)
    return out


@pytest.fixture(scope="module")
def auditemu(tmp_path_factory):
    """tests/hostemu/table_audit_emu.cpp: hs_table_audit's per-entry checks built for the host like the hostemu fixture's library."""
    lib = str(tmp_path_factory.mktemp("auditemu") / "libhs_auditemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "table_audit_emu.cpp")])
    emu = ctypes.CDLL(lib)
    emu.emu_comb_table_bytes.restype = ctypes.c_uint64
    return emu


def _table(emu, W, key):
    buf = ctypes.create_string_buffer(emu.emu_comb_table_bytes(W))
    assert emu.emu_build_comb_table(key, W, buf) == 1
    return bytearray(buf.raw)


def _audit(emu, W, table, key):
    win, ent = ctypes.c_int(-1), ctypes.c_int(-1)
    ok = emu.emu_table_audit(bytes(table), W, key, ctypes.byref(win), ctypes.byref(ent))
    return None if ok else (win.value, ent.value)


def _off(W, win, m, coord=0):
    return ((win * ((1 << (W - 1)) + 1)) + m) * ENTRY + 32 * coord


@pytest.fixture(scope="module", params=[8, 10])
def tables(request, hostemu, auditemu):
    W = request.param
    kx, ky = _valid_keys(hostemu, 2, 11 + W)
    return W, kx, ky, _table(auditemu, W, kx), _table(auditemu, W, ky), _table(auditemu, W, None)


def test_correct_key_and_base_tables_pass(auditemu, tables):
    W, kx, ky, tx, ty, tb = tables
    assert _audit(auditemu, W, tx, kx) is None
    assert _audit(auditemu, W, ty, ky) is None
    assert _audit(auditemu, W, tb, None) is None


@pytest.mark.parametrize("coord", [0, 1, 2])
@pytest.mark.parametrize("byte", [0, 13, 31])
def test_flipped_byte_is_found_at_its_entry(auditemu, tables, coord, byte):
    W, kx, _, tx, _, tb = tables
    H = 1 << (W - 1)
    for table, key in ((tx, kx), (tb, None)):
        for win, m in ((3, 5), (0, 1), (2, 1), (1, H), (0, 2)):
            t = bytearray(table)
            t[_off(W, win, m, coord) + byte] ^= 0x10
            assert _audit(auditemu, W, t, key) == (win, m), (win, m, coord, byte)


@pytest.mark.parametrize("coord", [0, 1, 2])
def test_non_canonical_twin_is_found(auditemu, tables, coord):
    W, kx, _, tx, _, _ = tables
    for win, m in ((2, 7), (0, 1), (5, 0)):
        t = bytearray(tx)
        o = _off(W, win, m, coord)
        v = int.from_bytes(t[o:o + 32], "little")
        t[o:o + 32] = (v + P).to_bytes(32, "little")
        assert _audit(auditemu, W, t, kx) == (win, m)


@pytest.mark.parametrize("a,b", [((1, 4), (1, 9)), ((0, 1), (0, 2)), ((2, 3), (5, 3)), ((3, 2), (3, 1))])
def test_swapped_entries_are_found_at_the_first(auditemu, tables, a, b):
    W, kx, _, tx, _, _ = tables
    t = bytearray(tx)
    oa, ob = _off(W, *a), _off(W, *b)
    t[oa:oa + ENTRY], t[ob:ob + ENTRY] = tx[ob:ob + ENTRY], tx[oa:oa + ENTRY]
    assert _audit(auditemu, W, t, kx) == min(a, b)


def test_altered_identity_entry_is_found(auditemu, tables):
    W, kx, _, tx, _, tb = tables
    for table, key in ((tx, kx), (tb, None)):
        for coord, byte in ((0, 0), (1, 5), (2, 0)):
            t = bytearray(table)
            t[_off(W, 4, 0, coord) + byte] ^= 1
            assert _audit(auditemu, W, t, key) == (4, 0)


@pytest.mark.parametrize("win", [0, 2])
def test_window_from_another_keys_table_breaks_the_link(auditemu, tables, win):
    W, kx, _, tx, ty, _ = tables
    t = bytearray(tx)
    lo, hi = _off(W, win, 0), _off(W, win + 1, 0)
    t[lo:hi] = ty[lo:hi]
    assert _audit(auditemu, W, t, kx) == (win, 1)


def test_correct_table_against_another_keys_bytes_breaks_the_anchor(auditemu, tables):
    W, kx, ky, tx, _, tb = tables
    assert _audit(auditemu, W, tx, ky) == (0, 1)
    assert _audit(auditemu, W, tb, kx) == (0, 1)
    assert _audit(auditemu, W, tx, None) == (0, 1)


# ---------------------------------------------------------------------------------------------------- wrappers
def test_cpp_wrapper_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "audit.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main() {\n"
                   "  hs::Engine e(0);\n"
                   "  std::vector<uint8_t> slot_bits;\n"
                   "  uint32_t f = e.table_audit(nullptr, nullptr, &slot_bits);\n"
                   "  std::vector<std::array<uint8_t, 32>> keys(e.key_slots());\n"
                   "  f |= e.table_audit(&keys, nullptr, nullptr);\n"
                   "  return (int)f;\n"
                   "}\n")
    exe = tmp_path / "audit"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert exe.exists()


def _strip(text):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", text, flags=re.S))


def test_rust_wrapper_audits_and_switches_the_gpu_off_on_a_finding():
    src = _strip(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    assert re.search(r"fn hs_table_audit\(ctx: \*mut HsCtx, expect_pks: \*const u8, expect_live: \*const u32, n_slots: usize, "
                     r"out_slot_bits: \*mut u8, out_failed: \*mut u32\) -> c_int;", src)
    body = re.search(r"pub fn audit_tables\(expected: &\[Option<\[u8; 32\]>\]\) -> Result<\(\), GpuError> \{(.*?)\n\}", src, flags=re.S)
    assert body, "gpu::audit_tables is missing"
    b = body.group(1)
    assert "hs_table_audit(" in b and "rc == HS_OK && failed == 0" in b
    assert "DISABLED.store(true, Ordering::Release)" in b
    # called after the start-up self-test and after every committee update
    st = re.search(r"pub fn self_test\(\).*?\n\}", src, flags=re.S).group(0)
    up = re.search(r"pub fn update_committee\(.*?\n\}", src, flags=re.S).group(0)
    assert "audit_tables(" in st and "audit_tables(" in up


# ---------------------------------------------------------------------------------------------------- GPU
HS_AUDIT_KEY, HS_AUDIT_FLAG, HS_AUDIT_LOOKUP, HS_AUDIT_TABLE, HS_AUDIT_BASE = 1, 2, 4, 8, 16


def _bad_keys(emu, n, seed):
    """Encodings that do not decompress (u/v is not a square), found with the host emulation."""
    rng = np.random.default_rng(seed)
    out, x, y = [], ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
    while len(out) < n:
        k = rng.bytes(32)
        if not emu.emu_decompress(k, x, y):
            out.append(np.frombuffer(k, np.uint8))
    return np.stack(out)


def _pubkeys(eng, n, seed):
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    return seeds, eng.keygen_batch(seeds)


def _live_bits(live):
    bm = np.zeros((len(live) + 31) // 32, np.uint32)
    for i, v in enumerate(live):
        if v:
            bm[i // 32] |= np.uint32(1 << (i % 32))
    return bm


def _expect_ok(eng, expect=None, live=None):
    failed, bits = eng.table_audit(expect, live)
    assert failed == 0, eng.last_error
    assert not bits.any()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 1000, 4096])
def test_registered_committees_pass(hostemu, n):
    from hotstuff_b200 import Engine
    eng = Engine(0)
    try:
        _, pks = _pubkeys(eng, n, 100 + n)
        pks = pks.copy()
        if n >= 1000:
            pks[5] = pks[3]  # a duplicated key: the hash table keeps the first
            pks[n - 10:n - 7] = _bad_keys(hostemu, 3, n)  # keys that do not decompress
        eng.committee_register(pks)
        assert eng.key_slots == n
        _expect_ok(eng)
        _expect_ok(eng, pks)
        _expect_ok(eng, pks, _live_bits([1] * n))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key_bits", [8, 10, 12, 13, 15, 17])
def test_forced_key_windows_pass(hostemu, key_bits):
    from hotstuff_b200 import Engine
    eng = Engine(0, key_window=key_bits)
    try:
        _, pks = _pubkeys(eng, 40, 7)
        pks = pks.copy()
        pks[7] = pks[2]
        pks[30:32] = _bad_keys(hostemu, 2, key_bits)
        eng.committee_register(pks)
        assert eng.window_bits[0] == key_bits
        _expect_ok(eng)
        _expect_ok(eng, pks)
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("base_bits", [16, 20, 24, 26])
def test_base_windows_pass(base_bits):
    from hotstuff_b200 import Engine
    eng = Engine(0, base_window=base_bits)
    try:
        assert eng.key_slots == 0
        _expect_ok(eng)  # a fresh context: the base table alone
        _, pks = _pubkeys(eng, 64, 9)
        eng.committee_register(pks)
        _expect_ok(eng, pks)
    finally:
        eng.close()


@pytest.mark.gpu
def test_committee_updates_pass_against_the_node_side_map():
    from hotstuff_b200 import Engine
    eng = Engine(0)
    try:
        _, pks = _pubkeys(eng, 200, 21)
        _, extra = _pubkeys(eng, 40, 22)
        eng.committee_register(pks)
        node = [bytes(k) for k in pks]  # index -> key, None = freed

        def update(add, remove):
            idx = eng.committee_update(np.frombuffer(b"".join(add), np.uint8).reshape(-1, 32) if add else None, remove)
            for i in remove:
                node[i] = None
            for k, i in zip(add, idx):
                while i >= len(node):
                    node.append(None)
                node[i] = bytes(k)
            assert eng.key_slots == len(node)
            exp = np.array([np.frombuffer(k, np.uint8) if k else np.zeros(32, np.uint8) for k in node], np.uint8)
            live = _live_bits([k is not None for k in node])
            _expect_ok(eng, exp, live)
            _expect_ok(eng)
            return exp, live

        update([], [3, 17, 150])                                           # removals
        update([bytes(extra[0]), bytes(extra[1])], [])                     # into freed slots
        update([bytes(extra[i]) for i in range(2, 12)], [5])               # freed slots, then 8 of the 16 spare slots
        update([bytes(pks[10]), bytes(extra[20]), bytes(extra[20])], [])   # a live key again; the same key twice in one call
        exp, live = update([bytes(extra[21])], [0, 1])
        # findings through the expectation: two swapped keys, a freed slot expected live, a live one expected freed
        sw = exp.copy()
        sw[[8, 9]] = sw[[9, 8]]
        failed, bits = eng.table_audit(sw, live)
        assert failed == HS_AUDIT_KEY and list(np.nonzero(bits)[0]) == [8, 9] and bits[8] == HS_AUDIT_KEY
        assert "slot 8" in eng.last_error and "KEY" in eng.last_error
        freed = [i for i, k in enumerate(node) if k is None][0]
        lv = [k is not None for k in node]
        lv[freed] = True
        failed, bits = eng.table_audit(exp, _live_bits(lv))
        assert failed == HS_AUDIT_KEY and list(np.nonzero(bits)[0]) == [freed]
        lv = [k is not None for k in node]
        lv[12] = False
        failed, bits = eng.table_audit(exp, _live_bits(lv))
        assert failed == HS_AUDIT_KEY and list(np.nonzero(bits)[0]) == [12]
        # an n_slots mismatch writes nothing
        from hotstuff_b200 import EngineError
        with pytest.raises(EngineError):
            eng.table_audit(exp[:-1], None)
    finally:
        eng.close()


@pytest.mark.gpu
def test_key_cache_tables_pass(oracle):
    from hotstuff_b200 import Engine, EngineError
    eng = Engine(0)
    try:
        _expect_ok(eng)
        seeds, pks = _pubkeys(eng, 96, 31)
        recs = _signed_recs(eng, seeds, pks, 512, 32)
        for _ in range(3):  # two passes over unknown keys (the keys are learned between calls)
            eng.verify_rec128(recs)
        n = eng.key_slots
        assert n == eng.cached_keys > 0
        _expect_ok(eng)
        with pytest.raises(EngineError):
            eng.table_audit(np.zeros((n, 32), np.uint8))
    finally:
        eng.close()


def _signed_recs(eng, seeds, pks, n, seed):
    rng = np.random.default_rng(seed)
    ki = rng.integers(0, len(pks), n).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    sig = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64] = sig
    recs[:, 64:96] = pks[ki]
    recs[:, 96:] = dig
    bad = rng.random(n) < 0.2
    recs[bad, 100] ^= 1
    return recs


@pytest.mark.gpu
def test_audit_is_read_only_and_leaves_a_vote_burst_alone(oracle):
    from hotstuff_b200 import Engine
    eng = Engine(0)
    try:
        seeds, pks = _pubkeys(eng, 4096, 41)
        eng.committee_register(pks)
        recs = _signed_recs(eng, seeds, pks, 3000, 42)
        want = oracle.verify_rec128(recs, mode=0)
        before = (eng.verify_rec128(recs, mode=0), eng.verify_rec128(recs, mode=1), eng.verify_rec128(recs[:40], mode=0))
        _expect_ok(eng, pks)
        after = (eng.verify_rec128(recs, mode=0), eng.verify_rec128(recs, mode=1), eng.verify_rec128(recs[:40], mode=0))
        for a, b in zip(before, after):
            assert np.array_equal(a, b)
        assert np.array_equal(before[0], want)

        def burst(q):
            votes = recs[:667]
            out = [None] * 667
            def worker(t):
                for i in range(t, 667, 16):
                    out[i] = q.wait(q.submit(votes[i:i + 1]))
            th = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
            for x in th:
                x.start()
            for x in th:
                x.join()
            st = q.stats()  # records per path; how many launches they shared depends on timing
            return np.array([bool(o[0]) for o in out], bool), {k: v for k, v in st.items() if not k.endswith("launches")}

        q1 = eng.queue()
        got1, st1 = burst(q1)
        q1.close()
        q2 = eng.queue()
        res = {}
        aud = threading.Thread(target=lambda: res.setdefault("a", eng.table_audit()))
        aud.start()
        got2, st2 = burst(q2)
        aud.join()
        q2.close()
        assert np.array_equal(got1, want[:667]) and np.array_equal(got2, want[:667])
        assert st1 == st2
        assert res["a"][0] == 0
    finally:
        eng.close()


@pytest.mark.gpu
def test_update_during_an_audit_ends_either_way_with_no_finding():
    from hotstuff_b200 import Engine, EngineError
    eng = Engine(0)
    try:
        _, pks = _pubkeys(eng, 4096, 51)
        _, extra = _pubkeys(eng, 8, 52)
        eng.committee_register(pks)
        outcomes = []
        for it in range(4):
            res = {}

            def audit():
                try:
                    res["r"] = eng.table_audit()
                except EngineError as e:
                    res["e"] = str(e)

            th = threading.Thread(target=audit)
            th.start()
            time.sleep(0.002 * it)
            eng.committee_update(extra[it:it + 1], [it])
            th.join()
            if "r" in res:
                assert res["r"][0] == 0
                outcomes.append("ok")
            else:
                assert "changed during the audit" in res["e"]
                outcomes.append("changed")
            _expect_ok(eng)
        assert len(outcomes) == 4
    finally:
        eng.close()
