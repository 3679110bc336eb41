"""hs_table_repair: the repair of what the table audit finds.

CPU: the test-only corruption hook is neither declared in the header nor exported by the product library; the C++ wrapper compiles and
links; the Rust shim repairs a finding before it can switch the GPU off.
GPU, on a build of the engine with the corruption hook (hs_test_poke, -DHS_TEST_HOOKS): real corrupt bytes in comb tables, key bytes,
flag bytes and the base-point table are found, repaired from the caller's map or the host mirror and proven by a clean audit, and the
repaired keys verify as the oracle does on every path; verification goes on beside a repair, and a repair empties the verify queues'
caches."""
import ctypes
import os
import re
import subprocess
import threading
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = 96  # bytes of one affine Niels entry
HS_AUDIT_KEY, HS_AUDIT_FLAG, HS_AUDIT_LOOKUP, HS_AUDIT_TABLE, HS_AUDIT_BASE = 1, 2, 4, 8, 16
POKE_TABLE, POKE_BASE, POKE_KEY, POKE_FLAG = 0, 1, 2, 3


def _strip(text):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", text, flags=re.S))


# ---------------------------------------------------------------------------------------------------- CPU
def test_corruption_hook_is_not_in_the_product():
    from hotstuff_b200 import build
    lib = build.build_engine()
    syms = subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    assert re.search(r"\bhs_table_repair\b", syms)
    assert not re.search(r"\bhs_test_poke\b", syms)
    assert "hs_test_poke" not in open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    src = open(os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")).read()
    hook = src[src.index("#ifdef HS_TEST_HOOKS"):]
    assert "extern \"C\" int hs_test_poke(" in hook[:hook.index("#endif")]


def test_cpp_wrapper_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "repair.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main() {\n"
                   "  hs::Engine e(0);\n"
                   "  std::vector<uint8_t> slot_bits;\n"
                   "  uint32_t found = 0;\n"
                   "  uint32_t f = e.table_repair(nullptr, nullptr, &found, &slot_bits);\n"
                   "  std::vector<std::array<uint8_t, 32>> keys(e.key_slots());\n"
                   "  f |= e.table_repair(&keys);\n"
                   "  return (int)(f | found);\n"
                   "}\n")
    exe = tmp_path / "repair"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert exe.exists()


def test_rust_wrapper_repairs_before_it_switches_the_gpu_off():
    src = _strip(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    assert re.search(r"fn hs_table_repair\(ctx: \*mut HsCtx, expect_pks: \*const u8, expect_live: \*const u32, n_slots: usize, "
                     r"out_slot_bits: \*mut u8, out_found: \*mut u32,\s*out_failed: \*mut u32\) -> c_int;", src)
    b = re.search(r"pub fn audit_tables\(expected: &\[Option<\[u8; 32\]>\]\) -> Result<\(\), GpuError> \{(.*?)\n\}", src, flags=re.S).group(1)
    audit, repair, off = b.index("hs_table_audit("), b.index("hs_table_repair("), b.index("DISABLED.store(true, Ordering::Release)")
    assert audit < repair < off
    # the GPU stays on when the repair succeeds: a return between the repair and the switch
    assert re.search(r"if rc == HS_OK \{ return Ok\(\(\)\); \}", b[repair:off])


# ---------------------------------------------------------------------------------------------------- GPU: the hook build
@pytest.fixture(scope="module")
def hooklib(tmp_path_factory):
    """The engine built with -DHS_TEST_HOOKS into a temporary directory, loaded next to the product library."""
    from hotstuff_b200 import _lib, build
    out = str(tmp_path_factory.mktemp("hook") / "libhs_crypto_hooks.so")
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
    subprocess.check_call([nvcc] + build.NVCC_FLAGS + ["-DHS_TEST_HOOKS", "-o", out] +
                          [os.path.join(build.CSRC, f) for f in ("hs_engine.cu", "hs_ingest.cpp", "hs_multi.cpp")], cwd=build.ROOT)
    lib = ctypes.CDLL(out)
    for name, (res, args) in _lib.SIGNATURES.items():
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    lib.hs_test_poke.restype = ctypes.c_int
    lib.hs_test_poke.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint8]
    return lib


def _engine(lib, base_window=0, key_window=0, key_cache=True):
    from hotstuff_b200 import Engine
    h = ctypes.c_void_p()
    rc = lib.hs_ctx_create(ctypes.byref(h), 0, (base_window & 0xff) | ((key_window & 0xff) << 8) | (0 if key_cache else 0x10000))
    assert rc == 0 and h
    e = Engine._view(lib, h, 0)
    e._owned = True
    return e


def _poke(eng, region, index, offset, mask=0x10):
    assert eng.lib.hs_test_poke(eng.h, region, index, offset, mask) == 0, eng.last_error


def _entry_off(W, win, m, byte=5):
    return ((win * ((1 << (W - 1)) + 1)) + m) * ENTRY + byte


def _windows(W):
    """Windows of a comb table of W-bit windows (sc_ndigits_rt)."""
    r = 253 % W
    return (253 + W - 1) // W + (1 if r in (0, W - 1) else 0)


def _last(W):
    """(window, entry) of the last entry of the last window."""
    return _windows(W) - 1, 1 << (W - 1)


def _keys(eng, n, seed):
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    return seeds, eng.keygen_batch(seeds)


def _golden_keys(golden):
    ref = golden["reference"]
    seeds = np.array([np.frombuffer(bytes.fromhex(s), np.uint8) for s in ref["seeds"]], np.uint8)
    pks = np.array([np.frombuffer(bytes.fromhex(p), np.uint8) for p in ref["pks"]], np.uint8)
    return seeds, pks


def _golden_recs(golden):
    """The golden file's reference records: the QC votes over qc_digest, key 3's signature over hello_digest and over bad_digest."""
    ref = golden["reference"]
    h = bytes.fromhex
    rows = [h(v["sig"]) + h(v["pk"]) + h(ref["qc_digest"]) for v in ref["qc_votes"]]
    for d in ("hello_digest", "bad_digest"):
        rows.append(h(ref["hello_sig_key3"]) + h(ref["pks"][3]) + h(ref[d]))
    return np.frombuffer(b"".join(rows), np.uint8).reshape(-1, 128).copy()


def _committee(eng, golden, n, seed):
    """n keys: the golden reference keys first, then seeded random ones (seeds kept, so every slot can sign)."""
    gs, gp = _golden_keys(golden)
    s, p = _keys(eng, n - len(gp), seed)
    return np.concatenate([gs, s]), np.concatenate([gp, p])


def _adversarial(eng, seeds, pks, slots, n, seed):
    """Records by the keys of `slots`: valid signatures, flipped bits in R, S and the digest, S + L, and records naming another key."""
    rng = np.random.default_rng(seed)
    ki = np.asarray(slots, np.uint32)[rng.integers(0, len(slots), n)]
    dig = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    sig = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = sig, pks[ki], dig
    kind = rng.integers(0, 6, n)
    for i in np.nonzero(kind == 1)[0]:
        recs[i, rng.integers(0, 32)] ^= 1 << rng.integers(0, 8)
    for i in np.nonzero(kind == 2)[0]:
        recs[i, 32 + rng.integers(0, 31)] ^= 1 << rng.integers(0, 8)
    for i in np.nonzero(kind == 3)[0]:
        recs[i, 96 + rng.integers(0, 32)] ^= 1 << rng.integers(0, 8)
    for i in np.nonzero(kind == 5)[0]:
        recs[i, 64:96] = pks[slots[(list(slots).index(ki[i]) + 1) % len(slots)]] if len(slots) > 1 else recs[i, 64:96]
    L = (1 << 252) + 27742317777372353535851937790883648493
    for i in np.nonzero(kind == 4)[0]:
        s = int.from_bytes(recs[i, 32:64].tobytes(), "little") + L
        if s < 1 << 256:
            recs[i, 32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
    return recs, ki


def _all_paths_match(eng, oracle, recs, ki):
    """Verdicts through key bytes (k_key_lookup + committee pass), committee indices, k_verify_small and k_verify_bulk equal the
    oracle's.  The committee-index records carry the slot's own key bytes."""
    want = oracle.verify_rec128(recs, mode=0)
    assert np.array_equal(eng.verify_rec128(recs, mode=0), want)
    byidx = recs.copy()
    byidx[:, 64:96] = eng._pks_for_test[ki]
    want_idx = oracle.verify_rec128(byidx, mode=0)
    assert np.array_equal(eng.verify_committee(ki, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(ki), dtype=np.uint32)), want_idx)
    for i in range(0, min(len(recs), 256), 64):
        assert np.array_equal(eng.verify_rec128(recs[i:i + 64], mode=0), want[i:i + 64])
    q = eng.queue()
    try:
        small = [q.wait(q.submit(recs[i:i + 1]))[0] for i in range(min(len(recs), 48))]
        assert np.array_equal(np.array(small, bool), want[:len(small)])
        grp = np.resize(recs, (1024, 128))  # a certificate of at least HS_QUEUE_BULK_MIN (1,002) committee records takes k_verify_bulk
        assert np.array_equal(q.wait(q.submit_group(grp)), np.resize(want, 1024))
        st = q.stats()
        assert st["small_launches"] > 0 and st["bulk_launches"] > 0, st
    finally:
        q.close()


def _expect_clean(eng, expect=None, live=None):
    failed, bits = eng.table_audit(expect, live)
    assert failed == 0, eng.last_error
    assert not bits.any()


def _live_bits(live):
    bm = np.zeros((len(live) + 31) // 32, np.uint32)
    for i, v in enumerate(live):
        if v:
            bm[i // 32] |= np.uint32(1 << (i % 32))
    return bm


@pytest.fixture
def big(hooklib, golden):
    """A 4 096-key committee at the window the budget picks (13 bits on an otherwise idle 80 GB H100).  One per test, released at its
    end: its tables take most of the device, and the tests with a forced key window need room for theirs."""
    eng = _engine(hooklib)
    seeds, pks = _committee(eng, golden, 4096, 61)
    assert eng.committee_register(pks).all()
    eng._pks_for_test = pks
    yield eng, seeds, pks
    eng.close()


@pytest.mark.gpu
def test_clean_context_is_an_audit_and_changes_nothing(big, oracle):
    eng, seeds, pks = big
    recs, ki = _adversarial(eng, seeds, pks, range(64), 256, 1)
    q = eng.queue()
    try:
        q.sig_cache(1 << 14)
        q.cert_cache(1 << 20)
        q.wait(q.submit_group(recs))
        launches = eng.kernel_launches
        before = (q.sig_stats(), q.cert_stats())
        found, failed, bits = eng.table_repair(pks)
        assert (found, failed) == (0, 0) and not bits.any()
        assert (q.sig_stats(), q.cert_stats()) == before
        assert eng.kernel_launches - launches == 3  # one audit: k_slot_audit and k_table_audit over the key and base tables
    finally:
        q.close()


def _table_case(eng, oracle, seeds, pks, W, slots, expect):
    """Pokes one entry in each of `slots` (window 0 entry 1, a middle window, the last entry of the last window, in turn), repairs,
    and checks the result."""
    mid = _windows(W) // 2
    spots = [(0, 1), (mid, 7), _last(W)]
    for k, s in enumerate(slots):
        _poke(eng, POKE_TABLE, s, _entry_off(W, *spots[k % 3], byte=k % 96))
    failed, _ = eng.table_audit()
    assert failed == HS_AUDIT_TABLE
    found, failed, bits = eng.table_repair(expect)
    assert failed == 0, eng.last_error
    assert found == HS_AUDIT_TABLE
    assert sorted(np.nonzero(bits)[0]) == sorted(slots) and set(bits[list(slots)]) == {HS_AUDIT_TABLE}
    _expect_clean(eng, pks)
    recs, ki = _adversarial(eng, seeds, pks, slots, 768, len(slots) + W)
    _all_paths_match(eng, oracle, recs, ki)


@pytest.mark.gpu
def test_table_entries_of_a_4096_key_committee(big, oracle, golden):
    eng, seeds, pks = big
    W = eng.window_bits[0]
    n_golden = len(golden["reference"]["pks"])
    _table_case(eng, oracle, seeds, pks, W, [3], pks)
    _table_case(eng, oracle, seeds, pks, W, list(range(n_golden)) + [100 + 37 * i for i in range(16 - n_golden)], None)
    g = _golden_recs(golden)
    assert np.array_equal(eng.verify_rec128(g), oracle.verify_rec128(g))


@pytest.mark.gpu
@pytest.mark.parametrize("key_bits", [8, 17])
def test_table_entries_at_forced_windows(hooklib, oracle, golden, key_bits):
    # A forced window does not shrink to the free memory, so the committee is kept small (24 keys and 16 spares: 3.8 GB at 17 bits)
    # and the base table narrow (16 bits), as other contexts of the session may hold device memory.
    eng = _engine(hooklib, base_window=16, key_window=key_bits)
    try:
        seeds, pks = _committee(eng, golden, 24, 70 + key_bits)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        assert eng.window_bits[0] == key_bits
        _table_case(eng, oracle, seeds, pks, key_bits, [5], pks)
        _table_case(eng, oracle, seeds, pks, key_bits, list(range(0, 24, 3)) + list(range(1, 24, 3)), None)
        g = _golden_recs(golden)
        assert np.array_equal(eng.verify_rec128(g), oracle.verify_rec128(g))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("authority", ["map", "mirror"])
def test_key_and_flag_bytes(hooklib, oracle, golden, authority):
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 200, 80)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        expect = pks if authority == "map" else None
        _poke(eng, POKE_FLAG, 9, 0, 0x01)
        _poke(eng, POKE_FLAG, 10, 0, 0x02)
        found, failed, bits = eng.table_repair(expect)
        assert failed == 0 and found & HS_AUDIT_FLAG and sorted(np.nonzero(bits)[0]) == [9, 10], eng.last_error
        _expect_clean(eng, pks)
        if authority == "map":
            # key bytes: the map restores them; the audit against the map names KEY
            _poke(eng, POKE_KEY, 20, 4)
            _poke(eng, POKE_KEY, 21, 31, 0x80)
            found, failed, bits = eng.table_repair(expect)
            assert failed == 0, eng.last_error
            assert found & HS_AUDIT_KEY and sorted(np.nonzero(bits)[0]) == [20, 21]
        else:
            # without a map the stored bytes cannot be told wrong, but their table no longer matches them: TABLE, rebuilt from the mirror
            _poke(eng, POKE_KEY, 20, 4)
            found, failed, bits = eng.table_repair(None)
            assert failed == 0, eng.last_error
            assert 20 in np.nonzero(bits)[0]
        _expect_clean(eng, pks)
        recs, ki = _adversarial(eng, seeds, pks, [9, 10, 20, 21], 512, 81)
        _all_paths_match(eng, oracle, recs, ki)
    finally:
        eng.close()


@pytest.mark.gpu
def test_the_map_is_the_authority(hooklib, oracle, golden):
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 100, 90)
        eng.committee_register(pks)
        new_seed, new_pk = _keys(eng, 1, 91)
        s, t = 40, 41
        node = pks.copy()
        node[s] = new_pk[0]
        live = [True] * 100
        live[t] = False
        lv = _live_bits(live)
        found, failed, bits = eng.table_repair(node, lv)
        assert failed == 0, eng.last_error
        assert found == HS_AUDIT_KEY and sorted(np.nonzero(bits)[0]) == [s, t]
        _expect_clean(eng, node, lv)
        # the new key verifies on the committee path at slot s; slot t rejects
        dig = np.frombuffer(np.random.default_rng(92).bytes(32 * 8), np.uint8).reshape(8, 32).copy()
        sig = eng.sign_digests(new_seed, new_pk, dig, key_idx=np.zeros(8, np.uint32))
        sig[3, 5] ^= 1
        recs = np.concatenate([sig, np.repeat(new_pk, 8, 0), dig], axis=1)
        want = oracle.verify_rec128(recs)
        assert np.array_equal(eng.verify_committee(np.full(8, s, np.uint32), sig, dig, msg_idx=np.arange(8, dtype=np.uint32)), want)
        assert np.array_equal(eng.verify_rec128(recs), want)
        assert not eng.verify_committee(np.full(8, t, np.uint32), sig, dig, msg_idx=np.arange(8, dtype=np.uint32)).any()
        # the old keys of s and t verify with correct verdicts on the generic path
        old, _ = _adversarial(eng, seeds, pks, [s, t], 300, 93)
        assert np.array_equal(eng.verify_rec128(old), oracle.verify_rec128(old))
        assert np.array_equal(eng.verify_rec128(old[:40]), oracle.verify_rec128(old[:40]))
    finally:
        eng.close()


@pytest.mark.gpu
def test_base_table(hooklib, oracle, golden):
    eng = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _committee(eng, golden, 64, 95)
        eng.committee_register(pks)
        eng._pks_for_test = pks
        wb = eng.window_bits[1]
        last_win, last_m = _last(wb)
        stride = (1 << (wb - 1)) + 1
        _poke(eng, POKE_BASE, 0 * stride + 1, 3)
        _poke(eng, POKE_BASE, last_win * stride + last_m, 70)
        failed, _ = eng.table_audit()
        assert failed == HS_AUDIT_BASE
        found, failed, bits = eng.table_repair(pks)
        assert (found, failed) == (HS_AUDIT_BASE, 0) and not bits.any(), eng.last_error
        _expect_clean(eng, pks)
        assert eng.self_test() == 0, eng.last_error
        recs, ki = _adversarial(eng, seeds, pks, range(64), 512, 96)
        _all_paths_match(eng, oracle, recs, ki)
    finally:
        eng.close()


@pytest.mark.gpu
def test_key_cache_table(hooklib, oracle):
    from hotstuff_b200 import EngineError
    eng = _engine(hooklib)
    try:
        seeds, pks = _keys(eng, 48, 97)
        recs, _ = _adversarial(eng, seeds, pks, range(48), 512, 98)
        for _ in range(3):  # the keys are learned between calls
            eng.verify_rec128(recs)
        n = eng.key_slots
        assert n == eng.cached_keys > 0
        W = eng.window_bits[0]
        _poke(eng, POKE_TABLE, n // 2, _entry_off(W, 1, 3))
        _poke(eng, POKE_FLAG, 0, 0, 0x02)
        found, failed, bits = eng.table_repair()
        assert failed == 0, eng.last_error
        assert found == HS_AUDIT_TABLE | HS_AUDIT_FLAG and sorted(np.nonzero(bits)[0]) == [0, n // 2]
        _expect_clean(eng)
        assert np.array_equal(eng.verify_rec128(recs), oracle.verify_rec128(recs))
        with pytest.raises(EngineError):
            eng.table_repair(np.zeros((n, 32), np.uint8))
    finally:
        eng.close()


def _burst(q, votes):
    out = [None] * len(votes)

    def worker(t):
        for i in range(t, len(votes), 16):
            out[i] = q.wait(q.submit(votes[i:i + 1]))

    th = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return np.array([bool(o[0]) for o in out], bool)


@pytest.mark.gpu
def test_verification_goes_on_beside_a_64_slot_repair(big, oracle):
    eng, seeds, pks = big
    W = eng.window_bits[0]
    slots = [64 * i + 5 for i in range(64)]
    votes, _ = _adversarial(eng, seeds, pks, list(range(4096)), 667, 99)
    votes[:200, 64:96] = pks[slots[:50]].repeat(4, 0)[:200]  # votes by keys under repair (re-signed below)
    rng = np.random.default_rng(100)
    dig = np.frombuffer(rng.bytes(32 * 200), np.uint8).reshape(200, 32).copy()
    ki = np.array(slots[:50], np.uint32).repeat(4)[:200]
    votes[:200, :64] = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    votes[:200, 96:] = dig
    votes[:200:7, 40] ^= 1
    want = oracle.verify_rec128(votes)
    # The top window's digit of a canonical scalar is at most 2^(253 - W (windows - 1)) + 1 (65 at 13 bits), so these entries are
    # never read by a verify: verdicts are exact before the repair takes the slots out, and any wrong verdict would come from the repair.
    top, H = _last(W)
    assert H - 64 > (1 << (253 - W * top)) + 1
    for k, s in enumerate(slots):
        _poke(eng, POKE_TABLE, s, _entry_off(W, top, H - k))
    q = eng.queue()
    try:
        res = {}
        th = threading.Thread(target=lambda: res.setdefault("r", eng.table_repair(pks)))
        th.start()
        got = [_burst(q, votes)]
        th.join()
        got.append(_burst(q, votes))
    finally:
        q.close()
    found, failed, bits = res["r"]
    assert failed == 0 and found == HS_AUDIT_TABLE and sorted(np.nonzero(bits)[0]) == slots
    for g in got:
        assert np.array_equal(g, want)
    _expect_clean(eng, pks)


@pytest.mark.gpu
def test_a_repair_empties_the_caches(big, oracle):
    eng, seeds, pks = big
    W = eng.window_bits[0]
    votes, _ = _adversarial(eng, seeds, pks, list(range(300)), 667, 101)
    want = oracle.verify_rec128(votes)
    q = eng.queue()
    try:
        q.sig_cache(1 << 14)
        q.cert_cache(1 << 20)
        dig = np.frombuffer(np.random.default_rng(102).bytes(32), np.uint8)
        qc_ki = np.arange(200, 300, dtype=np.uint32)
        qc = np.zeros((100, 128), np.uint8)
        qc[:, :64] = eng.sign_digests(seeds, pks, np.tile(dig, (100, 1)), key_idx=qc_ki)
        qc[:, 64:96], qc[:, 96:] = pks[qc_ki], dig
        assert q.wait(q.submit_group(qc, modes=np.ones(100, np.uint8))).all()
        assert np.array_equal(_burst(q, votes), want)
        assert q.sig_stats()["entries_held"] > 0 and q.cert_stats()["bytes_held"] > 0
        _poke(eng, POKE_TABLE, 7, _entry_off(W, 2, 9))
        found, failed, _ = eng.table_repair(pks)
        assert found == HS_AUDIT_TABLE and failed == 0, eng.last_error
        assert q.sig_stats()["entries_held"] == 0 and q.cert_stats()["bytes_held"] == 0
        assert np.array_equal(_burst(q, votes), want)
        assert q.wait(q.submit_group(qc, modes=np.ones(100, np.uint8))).all()
    finally:
        q.close()


@pytest.mark.gpu
def test_an_update_racing_a_repair_ends_with_a_clean_audit(hooklib, golden):
    from hotstuff_b200 import EngineError
    eng = _engine(hooklib)
    try:
        seeds, pks = _committee(eng, golden, 1000, 103)
        _, extra = _keys(eng, 8, 104)
        eng.committee_register(pks)
        W = eng.window_bits[0]
        node = [bytes(k) for k in pks]
        outcomes = []
        for it in range(4):
            for s in range(100 + 10 * it, 108 + 10 * it):
                _poke(eng, POKE_TABLE, s, _entry_off(W, 1, 2 + s))
            res = {}

            def repair():
                try:
                    res["r"] = eng.table_repair()
                except EngineError as e:
                    res["e"] = str(e)

            th = threading.Thread(target=repair)
            th.start()
            time.sleep(0.002 * it)
            idx = eng.committee_update(extra[it:it + 1], [it])
            th.join()
            node[it] = None
            for k, i in zip(extra[it:it + 1], idx):
                while i >= len(node):
                    node.append(None)
                node[i] = bytes(k)
            if "r" in res:
                assert res["r"][1] == 0, eng.last_error
                outcomes.append("ok")
            else:
                assert "changed during the repair" in res["e"] or "changed during the audit" in res["e"]
                outcomes.append("changed")
            exp = np.array([np.frombuffer(k, np.uint8) if k else np.zeros(32, np.uint8) for k in node], np.uint8)
            lv = _live_bits([k is not None for k in node])
            failed, bits = eng.table_audit(exp, lv)
            if failed:  # the repair lost the race before it began: its findings are still there, and a repair now clears them
                assert failed == HS_AUDIT_TABLE, eng.last_error
                assert eng.table_repair(exp, lv)[1] == 0, eng.last_error
            _expect_clean(eng, exp, lv)
        assert len(outcomes) == 4
    finally:
        eng.close()


@pytest.mark.gpu
def test_argument_errors_write_nothing(hooklib):
    from hotstuff_b200 import EngineError
    eng = _engine(hooklib)
    try:
        _, pks = _keys(eng, 40, 105)
        eng.committee_register(pks)
        found, failed = ctypes.c_uint32(77), ctypes.c_uint32(88)
        bits = np.full(40, 0xaa, np.uint8)
        lib = eng.lib
        for n in (39, 41):
            assert lib.hs_table_repair(eng.h, None, None, n, bits.ctypes.data_as(ctypes.c_void_p), ctypes.byref(found), ctypes.byref(failed)) == 2
        assert lib.hs_table_repair(eng.h, None, None, 40, None, None, ctypes.byref(failed)) == 2
        assert lib.hs_table_repair(eng.h, None, None, 40, None, ctypes.byref(found), None) == 2
        assert lib.hs_table_repair(None, None, None, 0, None, ctypes.byref(found), ctypes.byref(failed)) == 2
        assert (found.value, failed.value) == (77, 88) and (bits == 0xaa).all()
        with pytest.raises(EngineError):
            eng.table_repair(pks[:-1])
        # the hook range-checks every index
        for region, index, off in ((POKE_TABLE, 40, 0), (POKE_KEY, 0, 32), (POKE_FLAG, 0, 1), (POKE_BASE, 1 << 40, 0), (9, 0, 0)):
            assert lib.hs_test_poke(eng.h, region, index, off, 1) == 2
        _expect_clean(eng, pks)
    finally:
        eng.close()
