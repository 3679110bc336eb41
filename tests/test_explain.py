"""hs_explain_rec128: the table-free re-check that names every check of the decision procedure a record fails.

The expected mask of a record comes from the oracle's own primitives: S < l from Python integers, decompress_ok and is_small_order for A
and R, and HSO_EQ_OK of the oracle's verify for the equation.
CPU: explain_record under host emulation (tests/hostemu/explain_emu.cpp, compiled by this module) gives the expected mask on every golden
vector, adversarial records, every torsion encoding as A and as R, the edge values of S and seeded single-bit mutations of valid records;
the bit values agree across the header, Python and the Rust shim, and the shim explains only the first rejected record of a message.
GPU: k_explain gives the same masks at n = 1 and over several grid-stride rounds; the masks restate the verdicts of every verify path;
a false reject made by corrupting a live flag byte is told apart from a bad signature; the call reads no context state and changes none."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from oracle_api import EQ_OK, L_ORDER, make_adversarial, make_workload, to_rec128
from test_table_repair import POKE_FLAG, _engine, _keys, _poke, hooklib  # noqa: F401  (hooklib: the -DHS_TEST_HOOKS build, a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S_NONCANONICAL, A_INVALID, R_INVALID, A_SMALL, R_SMALL, EQUATION = 1, 2, 4, 8, 16, 32
PARSE = S_NONCANONICAL | A_INVALID | R_INVALID
SMALL = A_SMALL | R_SMALL
B_ENC = int("6666666666666666666666666666666666666666666666666666666666666658", 16).to_bytes(32, "little")


# ---------------------------------------------------------------------------------------------------- expected masks
class Expect:
    """Expected masks from the oracle's primitives; decompression results are cached per encoding (keys repeat)."""

    def __init__(self, oracle):
        self.o = oracle
        self.points = {}

    def point(self, enc, invalid, small):
        enc = bytes(enc)
        if enc not in self.points:
            ok = self.o.decompress_ok(enc)
            self.points[enc] = (not ok, ok and self.o.is_small_order(enc) == 1)
        bad, sm = self.points[enc]
        return (invalid if bad else 0) | (small if sm else 0)

    def parse(self, sig, pk):
        why = S_NONCANONICAL if int.from_bytes(bytes(sig[32:64]), "little") >= L_ORDER else 0
        return why | self.point(pk, A_INVALID, A_SMALL) | self.point(sig[:32], R_INVALID, R_SMALL)

    def one(self, sig, pk, msg):
        """Any message length: the equation from HSO_EQ_OK of the oracle's reference verify."""
        why = self.parse(sig, pk)
        if not why & PARSE and not self.o.flags(bytes(sig), bytes(pk), bytes(msg)) & EQ_OK:
            why |= EQUATION
        return why

    def recs(self, recs):
        """(n, 128) records: the equation from the oracle's batch-eq verdict, which is HSO_EQ_OK (the parse checks are in `why`)."""
        recs = np.ascontiguousarray(recs, np.uint8).reshape(-1, 128)
        eq = self.o.verify_rec128(recs, mode=1)
        out = np.zeros(len(recs), np.uint8)
        for i, r in enumerate(recs):
            why = self.parse(r[:64].tobytes(), r[64:96].tobytes())
            out[i] = why | (EQUATION if not why & PARSE and not eq[i] else 0)
        return out


def strict_ok(why):
    return np.asarray(why) == 0


def batch_ok(why):
    return (np.asarray(why) & (0xff & ~SMALL)) == 0


@pytest.fixture(scope="module")
def expect(oracle):
    return Expect(oracle)


# ---------------------------------------------------------------------------------------------------- record sets
def _rec(sig, pk, msg):
    return np.frombuffer(bytes(sig) + bytes(pk) + bytes(msg), np.uint8)


def _k(R, A, m):
    return int.from_bytes(hashlib.sha512(bytes(R) + bytes(A) + bytes(m)).digest(), "little") % L_ORDER


def torsion_records(oracle, golden, seed=3):
    """Every torsion encoding (the eight points, with their non-canonical and sign-bit twins) as A and as R: in place of a valid
    signature's A or R; every pair (A, R) with a random canonical S; A = T with R = [r]B, S = r over a message whose k kills T (the
    equation holds); A = T, R = -T, S = 0 over a message with k = 1 mod 8 (the equation holds with both small)."""
    rng = np.random.default_rng(seed)
    tors = [bytes.fromhex(t) for t in golden["torsion_encodings"]]
    seed_k = rng.bytes(32)
    pk = oracle.keygen(seed_k)
    rows = []
    for i in range(4):
        m = rng.bytes(32)
        sig = oracle.sign(seed_k, m)
        for t in tors:
            rows.append(_rec(sig, t, m))
            rows.append(_rec(t + sig[32:], pk, m))
    for ta in tors:
        for tr in tors:
            s = int(rng.integers(0, 2**62)) * int(rng.integers(1, 2**62)) % L_ORDER
            rows.append(_rec(tr + s.to_bytes(32, "little"), ta, rng.bytes(32)))
    for t in tors:
        r = int.from_bytes(rng.bytes(32), "little") % L_ORDER
        R = oracle.scalarmult(r, B_ENC)
        while True:
            m = rng.bytes(32)
            if _k(R, t, m) % 8 == 0:
                break
        rows.append(_rec(R + r.to_bytes(32, "little"), t, m))
        neg = bytearray(t)
        neg[31] ^= 0x80
        while True:
            m = rng.bytes(32)
            if _k(neg, t, m) % 8 == 1:
                break
        rows.append(_rec(bytes(neg) + bytes(32), t, m))
    return np.stack(rows)


def s_edge_records(oracle, seed=4):
    """Valid signatures with S replaced by l - 1, l and 2^256 - 1."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(4):
        sd, m = rng.bytes(32), rng.bytes(32)
        pk, sig = oracle.keygen(sd), oracle.sign(sd, m)
        rows.append(_rec(sig, pk, m))
        for s in (L_ORDER - 1, L_ORDER, 2**256 - 1):
            rows.append(_rec(sig[:32] + s.to_bytes(32, "little"), pk, m))
    return np.stack(rows)


def mutated_records(oracle, n, seed=5):
    """Seeded single-bit mutations of valid records (one bit anywhere in sig | pk | msg per record)."""
    w = make_workload(oracle, n, n_keys=64, seed=seed)
    recs = to_rec128(w)
    rng = np.random.default_rng(seed + 1)
    bits = rng.integers(0, 128 * 8, n)
    recs[np.arange(n), bits >> 3] ^= (1 << (bits & 7)).astype(np.uint8)
    return recs


def golden_rec128(golden):
    """The golden vectors with a 32-byte message, as packed records (the GPU call takes Digests)."""
    rows = [_rec(bytes.fromhex(v["sig"]), bytes.fromhex(v["pk"]), bytes.fromhex(v["msg"])) for v in golden["vectors"] if len(v["msg"]) == 64]
    return np.stack(rows)


# ---------------------------------------------------------------------------------------------------- CPU: host emulation
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("explain") / "libhs_explain.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "explain_emu.cpp")])
    lib = ctypes.CDLL(lib)
    lib.emu_explain.restype = None
    return lib


def emu_explain(emu, sigs, pks, msgs):
    n = len(sigs)
    sig = np.frombuffer(b"".join(bytes(s) for s in sigs), np.uint8).copy()
    pk = np.frombuffer(b"".join(bytes(p) for p in pks), np.uint8).copy()
    h = np.frombuffer(b"".join(hashlib.sha512(bytes(s[:32]) + bytes(p) + bytes(m)).digest() for s, p, m in zip(sigs, pks, msgs)), np.uint8).copy()
    out = np.zeros(n, np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    emu.emu_explain(vp(sig), vp(pk), vp(h), ctypes.c_size_t(n), vp(out))
    return out


def emu_explain_recs(emu, recs):
    return emu_explain(emu, [r[:64].tobytes() for r in recs], [r[64:96].tobytes() for r in recs], [r[96:].tobytes() for r in recs])


def _mismatches(got, want):
    bad = np.nonzero(np.asarray(got) != np.asarray(want))[0]
    return [(int(i), int(got[i]), int(want[i])) for i in bad[:8]]


def test_emu_golden_vectors(emu, expect, golden):
    vs = golden["vectors"]
    assert sum(v["group"] == "speccheck" for v in vs) == 12
    sigs, pks, msgs = ([bytes.fromhex(v[k]) for v in vs] for k in ("sig", "pk", "msg"))
    got = emu_explain(emu, sigs, pks, msgs)
    want = np.array([expect.one(s, p, m) for s, p, m in zip(sigs, pks, msgs)], np.uint8)
    assert not _mismatches(got, want), [(vs[i]["name"], g, w) for i, g, w in _mismatches(got, want)]
    # the masks restate the golden file's verdicts
    assert (strict_ok(got) == np.array([v["strict"] for v in vs])).all()
    assert (batch_ok(got) == np.array([v["batch_eq"] for v in vs])).all()
    for bit in (S_NONCANONICAL, A_INVALID, R_INVALID, A_SMALL, R_SMALL, EQUATION):
        assert (got & bit).any(), bit


def test_emu_adversarial_records(emu, expect, oracle):
    recs = make_adversarial(oracle, 1500, seed=11)
    got, want = emu_explain_recs(emu, recs), expect.recs(recs)
    assert not _mismatches(got, want), _mismatches(got, want)
    for bit in (S_NONCANONICAL, A_INVALID, R_INVALID, A_SMALL, R_SMALL, EQUATION):
        assert (got & bit).any(), bit


def test_emu_torsion_points_as_a_and_r(emu, expect, oracle, golden):
    recs = torsion_records(oracle, golden)
    got, want = emu_explain_recs(emu, recs), expect.recs(recs)
    assert not _mismatches(got, want), _mismatches(got, want)
    n_tors = len(golden["torsion_encodings"])
    tail = got[-2 * n_tors:]
    # every torsion A with a matching nonce verifies by the equation: small, never EQUATION; A = T, R = -T: both small
    assert (tail[0::2] == A_SMALL).all() and (tail[1::2] == A_SMALL | R_SMALL).all(), tail


def test_emu_s_edge_values(emu, expect, oracle):
    recs = s_edge_records(oracle)
    got, want = emu_explain_recs(emu, recs), expect.recs(recs)
    assert not _mismatches(got, want), _mismatches(got, want)
    assert list(got[:4]) == [0, EQUATION, S_NONCANONICAL, S_NONCANONICAL]


def test_emu_single_bit_mutations(emu, expect, oracle):
    recs = mutated_records(oracle, 3000)
    got, want = emu_explain_recs(emu, recs), expect.recs(recs)
    assert not _mismatches(got, want), _mismatches(got, want)


# ---------------------------------------------------------------------------------------------------- CPU: bindings
def _strip(text):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", text, flags=re.S))


def test_bits_agree_across_header_python_and_rust():
    from hotstuff_b200 import engine
    hdr = open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    rs = _strip(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    names = ("S_NONCANONICAL", "A_INVALID", "R_INVALID", "A_SMALL", "R_SMALL", "EQUATION")
    for name, bit in zip(names, (S_NONCANONICAL, A_INVALID, R_INVALID, A_SMALL, R_SMALL, EQUATION)):
        assert re.search(r"#define HS_WHY_%s %du\b" % (name, bit), hdr), name
        assert getattr(engine, "WHY_" + name) == bit
        assert "pub const HS_WHY_%s: u8 = %d;" % (name, bit) in rs
    assert re.search(r"int hs_explain_rec128\(hs_ctx \*ctx, const hs_rec128 \*recs, size_t n, uint8_t \*out_why", hdr)


def test_rust_helper_explains_only_the_first_rejected_record():
    src = _strip(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    body = re.search(r"pub fn explain_rejected\(recs: &\[HsRec128\], modes: &\[u8\], verdicts: &\[bool\]\) -> Option<Explained> \{(.*?)\n\}",
                     src, flags=re.S).group(1)
    assert "verdicts.iter().position(|ok| !ok)?" in body
    assert "hs_explain_rec128(c, &recs[index], 1, &mut why)" in body
    assert "if rc != HS_OK { return None; }" in body
    # a fault is a record the re-check finds valid in its own mode
    assert "why & !(HS_WHY_A_SMALL | HS_WHY_R_SMALL) == 0" in body and "why == 0" in body


CPP_MAIN = r'''#include <cstdio>
#include <vector>
#include "hs_crypto.hpp"
int main(int argc, char **argv) {
  FILE *f = std::fopen(argv[1], "rb");
  std::vector<hs_rec128> recs;
  hs_rec128 r;
  while (std::fread(&r, sizeof r, 1, f) == 1) recs.push_back(r);
  std::fclose(f);
  hs::Engine e(0);
  const std::vector<uint8_t> why = e.explain(recs.data(), recs.size());
  f = std::fopen(argv[2], "wb");
  std::fwrite(why.data(), 1, why.size(), f);
  std::fclose(f);
  return 0;
}
'''


@pytest.fixture(scope="module")
def cpp_explain(tmp_path_factory):
    from hotstuff_b200 import build
    lib = build.build_engine()
    d = tmp_path_factory.mktemp("explain_cpp")
    (d / "explain.cpp").write_text(CPP_MAIN)
    exe = d / "explain"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(d / "explain.cpp"), "-o", str(exe), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def test_cpp_wrapper_compiles_and_links(cpp_explain):
    assert cpp_explain.exists()


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine, build
    build.build_engine()
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def seeded(oracle):
    """2^16 seeded records over 256 keys, 1 % of them with one flipped bit."""
    w = make_workload(oracle, 1 << 16, n_keys=256, seed=21, corrupt_frac=0.01)
    return w, to_rec128(w)


@pytest.fixture(scope="module")
def sets(oracle, golden, expect, seeded):
    """name -> (records, expected masks)."""
    out = {}
    for name, recs in (("golden", golden_rec128(golden)), ("adversarial", make_adversarial(oracle, 2000, seed=12)),
                       ("torsion", torsion_records(oracle, golden)), ("s_edges", s_edge_records(oracle)),
                       ("mutations", mutated_records(oracle, 3000)), ("seeded", seeded[1])):
        out[name] = (recs, expect.recs(recs))
    return out


@pytest.mark.gpu
def test_kernel_matches_the_oracle(ctx, sets):
    for name, (recs, want) in sets.items():
        got = ctx.explain(recs)
        assert got.dtype == np.uint8 and got.shape == want.shape
        assert not _mismatches(got, want), (name, _mismatches(got, want))
        for i in range(0, len(recs), max(1, len(recs) // 12)):  # n = 1
            assert int(ctx.explain(recs[i:i + 1])[0]) == int(want[i]), (name, i)


@pytest.mark.gpu
def test_kernel_over_several_grid_stride_rounds(ctx, sets):
    # 2^18 records: a launch has at most 4 blocks of 128 threads per SM (67,584 threads on a 132-SM H100), so each thread takes several
    recs, want = sets["seeded"]
    big = np.concatenate([sets["adversarial"][0], np.tile(recs, (4, 1))])
    got = ctx.explain(big)
    want = np.concatenate([sets["adversarial"][1], np.tile(want, 4)])
    assert not _mismatches(got, want), _mismatches(got, want)


def _all_records(sets):
    recs = np.concatenate([sets[k][0] for k in ("golden", "adversarial", "seeded")])
    return recs, np.concatenate([sets[k][1] for k in ("golden", "adversarial", "seeded")])


def _check_identities(e, recs, why, what):
    for mode, ok in ((0, strict_ok(why)), (1, batch_ok(why))):
        got = e.verify_rec128(recs, mode)
        assert (got == ok).all(), (what, mode, np.nonzero(got != ok)[0][:8])


@pytest.mark.gpu
def test_identities_hold_against_hs_verify_rec128(ctx, sets, seeded, golden):
    from hotstuff_b200 import Engine
    recs, why = _all_records(sets)
    assert (ctx.explain(recs) == why).all()
    _check_identities(ctx, recs, why, "default context")
    # keys in and out of a registered committee: half of the seeded keys, plus the golden reference keys
    pks = seeded[0]["pks"]
    ref = np.array([np.frombuffer(bytes.fromhex(p), np.uint8) for p in golden["reference"]["pks"]], np.uint8)
    committee = np.concatenate([pks[: len(pks) // 2], ref])
    members = {p.tobytes() for p in committee}
    latency = np.array([i for i, r in enumerate(recs) if r[64:96].tobytes() in members][:48])  # n <= 64, every key registered
    for kw in (0, 8, 16):
        e = Engine(0, base_window=16 if kw else 0, key_window=kw)
        try:
            _check_identities(e, recs, why, "no committee, key window %d" % kw)
            e.committee_register(committee)
            _check_identities(e, recs, why, "committee, key window %d" % kw)
            _check_identities(e, recs[latency], why[latency], "committee latency path, key window %d" % kw)
        finally:
            e.close()


@pytest.mark.gpu
def test_identities_hold_against_the_queue_small_and_bulk_kernels(sets, seeded):
    from hotstuff_b200 import Engine
    w, recs = seeded
    why = sets["seeded"][1]
    e = Engine(0)
    try:
        e.committee_register(w["pks"])
        members = {p.tobytes() for p in w["pks"]}
        inside = np.array([i for i, r in enumerate(recs) if r[64:96].tobytes() in members])  # the queue's device path
        rng = np.random.default_rng(31)
        q = e.queue(8192)
        for n in (64, 700, 3000):  # small launches below 1,002 records, a bulk launch above
            pick = rng.choice(inside, n, replace=False)
            modes = rng.integers(0, 2, n).astype(np.uint8)
            got = q.wait(q.submit_group(recs[pick], modes))
            want = np.where(modes == 1, batch_ok(why[pick]), strict_ok(why[pick]))
            assert (np.asarray(got) == want).all(), (n, np.nonzero(np.asarray(got) != want)[0][:8])
        st = q.stats()
        assert st["small_launches"] >= 2 and st["bulk_launches"] >= 1 and st["slow_requests"] == 0, st
    finally:
        e.close()


@pytest.mark.gpu
def test_identities_hold_against_hs_verify_groups_with_mixed_modes(ctx, oracle, expect, sets, seeded):
    # items over 32-byte preimages: their Digests are the messages the explained records carry
    w, _ = seeded
    n_valid = 4096
    rng = np.random.default_rng(41)
    pre = rng.integers(0, 256, (n_valid, 32), dtype=np.uint8)
    dig = np.stack([np.frombuffer(hashlib.sha512(p.tobytes()).digest()[:32], np.uint8) for p in pre])
    ki = rng.integers(0, len(w["pks"]), n_valid).astype(np.uint32)
    sig = oracle.sign_batch(w["seeds"], w["pks"], ki, dig.reshape(-1), np.arange(n_valid + 1, dtype=np.uint64) * 32)
    pk = w["pks"][ki].copy()
    flip = rng.choice(n_valid, 41, replace=False)
    sig[flip[:20], rng.integers(0, 64, 20)] ^= 4
    pk[flip[20:], rng.integers(0, 32, 21)] ^= 1
    adv = sets["adversarial"][0]
    adv_dig = np.stack([np.frombuffer(hashlib.sha512(m.tobytes()).digest()[:32], np.uint8) for m in adv[:, 96:]])
    pre = np.concatenate([pre, adv[:, 96:]])
    sig = np.concatenate([sig, adv[:, :64]])
    pk = np.concatenate([pk, adv[:, 64:96]])
    recs = np.concatenate([sig, pk, np.concatenate([dig, adv_dig])], axis=1)
    why = ctx.explain(recs)
    assert (why == expect.recs(recs)).all()
    n = len(recs)
    modes = rng.integers(0, 2, n).astype(np.uint8)
    groups = rng.integers(0, 512, n).astype(np.uint32)
    _, items = ctx.verify_groups(pre.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 32, sig, np.arange(n, dtype=np.uint32), groups, 512,
                                 mode=modes, pk=pk, want_items=True)
    want = np.where(modes == 1, batch_ok(why), strict_ok(why))
    assert (items == want).all(), np.nonzero(items != want)[0][:8]


@pytest.mark.gpu
def test_a_corrupt_flag_byte_is_a_false_reject_the_explanation_exposes(ctx, oracle, hooklib):
    e = _engine(hooklib, base_window=16)
    try:
        seeds, pks = _keys(e, 32, seed=51)
        assert e.committee_register(pks).all()
        ki = np.arange(128, dtype=np.uint32) % 32
        msgs = np.random.default_rng(52).integers(0, 256, (128, 32), dtype=np.uint8)
        sig = oracle.sign_batch(seeds, pks, ki, msgs.reshape(-1), np.arange(129, dtype=np.uint64) * 32)
        recs = np.concatenate([sig, pks[ki], msgs], axis=1)
        assert e.verify_rec128(recs).all()
        _poke(e, POKE_FLAG, 7, 0, 0x01)  # slot 7's key now reads as "does not decompress": its valid signatures are rejected
        got = e.verify_rec128(recs)
        assert (got == (ki != 7)).all()
        why = e.explain(recs)
        assert (why == 0).all()  # every rejected record is valid: the disagreement names an engine fault
        found, failed, slot_bits = e.table_repair(expect=pks)
        assert failed == 0 and found and slot_bits[7]
        assert e.verify_rec128(recs).all() and (e.explain(recs) == 0).all()
    finally:
        e.close()


@pytest.mark.gpu
def test_explaining_reads_and_changes_no_context_state(oracle, sets):
    from hotstuff_b200 import Engine
    recs, why = sets["adversarial"]
    e = Engine(0)  # key cache on, no committee
    try:
        w = make_workload(oracle, 256, n_keys=16, seed=61)
        e.committee_register(w["pks"])
        q = e.queue()
        t = q.wait(q.submit_group(to_rec128(w)[:64]))
        assert np.asarray(t).all()
        stats, launches = q.stats(), e.kernel_launches
        for n in (1, 100, len(recs)):
            assert (e.explain(recs[:n]) == why[:n]).all()
            assert e.kernel_launches == launches + 1
            launches = e.kernel_launches
        assert q.stats() == stats
        assert (e.explain(np.zeros((0, 128), np.uint8)) == np.zeros(0, np.uint8)).all() and e.kernel_launches == launches
    finally:
        e.close()
    e = Engine(0)  # key cache on: a verify call parks the keys it has no table for, and the next call builds their tables
    try:
        known = to_rec128(make_workload(oracle, 256, n_keys=16, seed=62))
        e.verify_rec128(known)
        e.verify_rec128(known)
        cached = e.cached_keys
        assert cached > 0
        for _ in range(2):
            assert (e.explain(recs) == why).all()  # keys the cache has never seen
        assert e.cached_keys == cached
        e.verify_rec128(known)  # would build tables for keys parked by the calls before it
        assert e.cached_keys == cached
    finally:
        e.close()


@pytest.mark.gpu
def test_argument_errors_write_nothing(ctx):
    lib = ctx.lib
    out = np.full(4, 0xAB, np.uint8)
    recs = np.zeros((4, 128), np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert lib.hs_explain_rec128(ctx.h, None, 4, vp(out)) == 2
    assert lib.hs_explain_rec128(ctx.h, vp(recs), 4, None) == 2
    assert lib.hs_explain_rec128(None, vp(recs), 4, vp(out)) == 2
    assert "hs_explain_rec128" in ctx.last_error
    assert (out == 0xAB).all()
    assert lib.hs_explain_rec128(ctx.h, None, 0, None) == 0 and (out == 0xAB).all()


@pytest.mark.gpu
def test_cpp_binding_gives_the_same_masks(ctx, cpp_explain, sets, tmp_path):
    recs, _ = sets["adversarial"]
    (tmp_path / "recs.bin").write_bytes(recs.tobytes())
    subprocess.check_call([str(cpp_explain), str(tmp_path / "recs.bin"), str(tmp_path / "why.bin")])
    got = np.frombuffer((tmp_path / "why.bin").read_bytes(), np.uint8)
    assert (got == ctx.explain(recs)).all()
