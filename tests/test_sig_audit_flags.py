"""flags_from_why (verify_core.cuh): the flag byte the verify paths' verify_flags_from writes, derived from explain_record's table-free
mask.  The signature cache's audit (k_sig_audit) trusts this rule to re-derive a stored entry's flags from its 128 bytes, so it is pinned
here under host emulation, byte for byte against the generic-key and committee-key verify paths, before any GPU runs it:
the golden vectors (the 12 speccheck classes included), the edge-digit fixture, every torsion encoding as A and as R, S at its edges,
and a few thousand seeded adversarial records (bit flips in R, S, A and M; small-order and non-decompressing R and A; S >= l)."""
import ctypes
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from oracle_api import L_ORDER, make_adversarial, make_workload, to_rec128
from test_explain import s_edge_records, torsion_records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F_PARSE_OK, F_EQ, F_SMALL, F_STRICT = 1, 4, 8, 16
S_NONCANONICAL, A_INVALID, R_INVALID, A_SMALL, R_SMALL, EQUATION = 1, 2, 4, 8, 16, 32


@pytest.fixture(scope="module")
def audit_emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("sig_audit") / "libhs_sig_audit_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "sig_audit_emu.cpp")])
    lib = ctypes.CDLL(lib)
    lib.emu_flags_from_why.restype = ctypes.c_uint32
    lib.emu_flags_from_why.argtypes = [ctypes.c_uint32]
    lib.emu_audit_flags.restype = None
    return lib


def audit_flags(lib, sigs, pks, msgs):
    """flags_from_why(explain_record(..)) per record, any message length (h = SHA-512(R || A || msg) is hashed here)."""
    n = len(sigs)
    sig = np.frombuffer(b"".join(bytes(s) for s in sigs), np.uint8).copy()
    pk = np.frombuffer(b"".join(bytes(p) for p in pks), np.uint8).copy()
    h = np.frombuffer(b"".join(hashlib.sha512(bytes(s[:32]) + bytes(p) + bytes(m)).digest() for s, p, m in zip(sigs, pks, msgs)), np.uint8).copy()
    out = np.zeros(n, np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    lib.emu_audit_flags(vp(sig), vp(pk), vp(h), ctypes.c_size_t(n), vp(out))
    return out


def verify_flags(hostemu, fn, sigs, pks, msgs):
    f = getattr(hostemu, fn)
    return np.array([f(bytes(s), bytes(p), bytes(m), ctypes.c_uint64(len(m))) for s, p, m in zip(sigs, pks, msgs)], np.uint8)


def split(recs):
    recs = np.ascontiguousarray(recs, np.uint8).reshape(-1, 128)
    return [r[:64].tobytes() for r in recs], [r[64:96].tobytes() for r in recs], [r[96:].tobytes() for r in recs]


def check(audit_emu, hostemu, sigs, pks, msgs, paths=("emu_verify_generic", "emu_verify_committee")):
    got = audit_flags(audit_emu, sigs, pks, msgs)
    for fn in paths:
        want = verify_flags(hostemu, fn, sigs, pks, msgs)
        bad = np.nonzero(got != want)[0]
        assert not len(bad), (fn, [(int(i), int(got[i]), int(want[i])) for i in bad[:8]])
    return got


def flipped_records(oracle, n, seed):
    """Seeded adversarial records built from valid signatures: one bit flipped in R, S, A or M; R or A replaced by a small-order
    encoding or by bytes that do not decompress; S replaced by S + l or a value >= l."""
    rng = np.random.default_rng(seed)
    recs = to_rec128(make_workload(oracle, n, n_keys=32, seed=seed))
    Y8 = 0x05fc536d880238b13933c6d305acdfd5f098eff289f4c345b027b2c28f95e826
    P = 2**255 - 19
    tors = [(y | (s << 255)).to_bytes(32, "little") for y in (0, 1, P - 1, P + 1, Y8, P - Y8) for s in (0, 1)]
    kind = rng.integers(0, 8, n)
    for i in range(n):
        k = int(kind[i])
        if k < 4:  # a bit of R (0), S (1), A (2) or M (3)
            b = int(rng.integers(0, 256))
            recs[i, 32 * k + (b >> 3)] ^= 1 << (b & 7)
        elif k == 4:  # small-order R or A
            off = (0, 64)[int(rng.integers(0, 2))]
            recs[i, off:off + 32] = np.frombuffer(tors[int(rng.integers(0, len(tors)))], np.uint8)
        elif k == 5:  # R or A that does not decompress (y with no square root: retried until the oracle says so)
            off = (0, 64)[int(rng.integers(0, 2))]
            while True:
                enc = rng.bytes(32)
                if not oracle.decompress_ok(enc):
                    break
            recs[i, off:off + 32] = np.frombuffer(enc, np.uint8)
        elif k == 6:  # S + l when it fits, else S with its top bits set
            s = int.from_bytes(recs[i, 32:64].tobytes(), "little")
            s = s + L_ORDER if s + L_ORDER < 2**256 else s | (7 << 253)
            recs[i, 32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
        else:  # S >= l drawn at random
            s = int(rng.integers(0, 2**62)) * (2**194) % (2**256 - L_ORDER) + L_ORDER
            recs[i, 32:64] = np.frombuffer(s.to_bytes(32, "little"), np.uint8)
    return recs


def test_rule_restates_both_verdicts(audit_emu):
    for why in range(64):
        f = audit_emu.emu_flags_from_why(why)
        assert bool(f & F_STRICT) == (why == 0)
        assert bool(f & F_EQ) == (why & ~(A_SMALL | R_SMALL) == 0)
        assert bool(f & F_SMALL) == bool(why & (A_SMALL | R_SMALL))
        assert bool(f & F_PARSE_OK) == (not why & (S_NONCANONICAL | A_INVALID))
        assert not f & ~(F_PARSE_OK | F_EQ | F_SMALL | F_STRICT)


def test_golden_vectors(audit_emu, hostemu, golden):
    vs = golden["vectors"]
    assert len(vs) == 151 and sum(v["group"] == "speccheck" for v in vs) == 12
    sigs, pks, msgs = ([bytes.fromhex(v[k]) for v in vs] for k in ("sig", "pk", "msg"))
    got = check(audit_emu, hostemu, sigs, pks, msgs)
    assert ((got & F_STRICT) != 0).tolist() == [bool(v["strict"]) for v in vs]
    assert ((got & F_EQ) != 0).tolist() == [bool(v["batch_eq"]) for v in vs]
    # every flag combination the verify paths write for these vectors, so the rule is tested on each
    assert {0, F_PARSE_OK, F_PARSE_OK | F_EQ | F_STRICT, F_PARSE_OK | F_EQ | F_SMALL} <= set(got.tolist())


def test_edge_digit_fixture(audit_emu, hostemu):
    with open(os.path.join(ROOT, "tests", "golden", "edge_digits.json")) as f:
        recs = json.load(f)["records"]
    sigs, pks, msgs = ([bytes.fromhex(r[k]) for r in recs] for k in ("sig", "pk", "msg"))
    got = check(audit_emu, hostemu, sigs, pks, msgs)
    assert (got == F_PARSE_OK | F_EQ | F_STRICT).all()


def test_torsion_and_s_edges(audit_emu, hostemu, oracle, golden):
    recs = np.concatenate([torsion_records(oracle, golden), s_edge_records(oracle)])
    got = check(audit_emu, hostemu, *split(recs))
    assert (got == F_PARSE_OK | F_EQ | F_SMALL).any()


def test_seeded_adversarial_generic_key(audit_emu, hostemu, oracle):
    recs = np.concatenate([make_adversarial(oracle, 1500, seed=21), flipped_records(oracle, 2000, seed=22)])
    got = check(audit_emu, hostemu, *split(recs), paths=("emu_verify_generic",))
    for f in (0, F_PARSE_OK, F_PARSE_OK | F_EQ | F_STRICT, F_PARSE_OK | F_EQ | F_SMALL, F_PARSE_OK | F_SMALL):
        assert (got == f).any(), f


def test_seeded_adversarial_committee_key(audit_emu, hostemu, oracle):
    """The committee path builds the key's comb table per record under emulation, so it takes a sample of both generators."""
    recs = np.concatenate([make_adversarial(oracle, 150, seed=23), flipped_records(oracle, 250, seed=24)])
    got = check(audit_emu, hostemu, *split(recs))
    assert (got == F_PARSE_OK | F_EQ | F_SMALL).any() and (got == F_PARSE_OK | F_EQ | F_STRICT).any()
