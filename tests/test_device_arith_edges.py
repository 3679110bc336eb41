"""The device field and scalar arithmetic at the paths random data does not reach, and signatures whose comb digits reach the extreme
entries of a window.

Field elements are 8 saturated 32-bit limbs, any value in [0, 2^256).  fe_mul / fe_sqr / fe_add / fe_sub (generated PTX,
hotstuff_b200/csrc/fe_asm.cuh) end in an out-of-line path: the ripple, taken when the last +38 fold carries (or the -38 borrows) out of
limb 0, and inside it a second wrap when limbs 1..7 pass the carry all the way out.  Random products take the ripple about once in 10^7
and the second wrap never, so these tests build inputs that do, and hold every primitive to a model that is exact about the bits, not
just right mod p (T = 2^256):
  mul / sqr   v1 = L + 38 H (the 512-bit product is H T + L);  s = (v1 mod T) + 38 floor(v1 / T);  r = (s mod T) + 38 floor(s / T)
  add         the same two folds of v1 = a + b
  sub         d = a - b;  while d < 0 (at most twice): d += T - 38
The model also names the path each input takes, and every input class asserts a minimum count of its path, so no class can silently
become empty.  CPU: the generator reproduces fe_asm.cuh byte for byte (and proves the same paths in its simulator), the host emulation
equals the models bit for bit, the harness compiles for sm_90a, and the edge-digit fixture makes every claim it lists.  GPU: the
harness (tests/cuda/arith_harness.cu, the same inlines the kernels run) equals the models, the host emulation and Python integers; the
edge-digit records pass every verify path of hs_self_test at every key width 8..17 and base widths 16, 20 and 24."""
import ctypes
import hashlib
import importlib.util
import json
import os
import random
import re
import subprocess

import numpy as np
import pytest

from oracle_api import L_ORDER, P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "cuda", "arith_harness.cu")
EDGE = os.path.join(ROOT, "tests", "golden", "edge_digits.json")
T = 1 << 256
M = 2 * P  # = T - 38
M32 = (1 << 32) - 1
MUL, SQR, ADD, SUB, CANON, INVERT, POW_P58, NEG, IS_ZERO, EQ, IS_NEG, SQR_N = range(12)


# ---------------------------------------------------------------------------------------------------- bit-exact models
def _fold2(v1):
    s = v1 % T + 38 * (v1 >> 256)
    return s % T + 38 * (s >> 256)


def m_mul(a, b):
    ab = a * b
    return _fold2(ab % T + 38 * (ab >> 256))


def m_sqr(a):
    return m_mul(a, a)


def m_add(a, b):
    return _fold2(a + b)


def m_sub(a, b):
    d = a - b
    for _ in range(2):
        if d < 0:
            d += T - 38
    return d


def m_sqr_n(a, n):
    r = m_sqr(a)
    for _ in range(1, n):
        r = m_sqr(r)
    return r


def _m_pow2_250_1(z):
    """fe_pow2_250_1, step for step: (z^(2^250 - 1), z^11)."""
    z2 = m_sqr(z)
    z9 = m_mul(m_sqr_n(z2, 2), z)
    z11 = m_mul(z9, z2)
    a = m_mul(m_sqr(z11), z9)
    b = m_mul(m_sqr_n(a, 5), a)
    c = m_mul(m_sqr_n(b, 10), b)
    t = m_mul(m_sqr_n(c, 20), c)
    b = m_mul(m_sqr_n(t, 10), b)
    c = m_mul(m_sqr_n(b, 50), b)
    t = m_mul(m_sqr_n(c, 100), c)
    return m_mul(m_sqr_n(t, 50), b), z11


def m_invert(z):
    t, z11 = _m_pow2_250_1(z)
    return m_mul(m_sqr_n(t, 5), z11)


def m_pow_p58(z):
    t, _ = _m_pow2_250_1(z)
    return m_mul(m_sqr_n(t, 2), z)


def model(op, a, b):
    return {MUL: lambda: m_mul(a, b), SQR: lambda: m_sqr(a), ADD: lambda: m_add(a, b), SUB: lambda: m_sub(a, b), CANON: lambda: a % P,
            INVERT: lambda: m_invert(a), POW_P58: lambda: m_pow_p58(a), NEG: lambda: m_sub(0, a), IS_ZERO: lambda: int(a % P == 0),
            EQ: lambda: int((a - b) % P == 0), IS_NEG: lambda: (a % P) & 1, SQR_N: lambda: m_sqr_n(a, b)}[op]()


def truth(op, a, b):
    """The value mod p (or the predicate) from Python integers alone: what any correct representation must reduce to."""
    return {MUL: lambda: a * b % P, SQR: lambda: a * a % P, ADD: lambda: (a + b) % P, SUB: lambda: (a - b) % P, CANON: lambda: a % P,
            INVERT: lambda: pow(a, P - 2, P), POW_P58: lambda: pow(a, (P - 5) // 8, P), NEG: lambda: -a % P, IS_ZERO: lambda: int(a % P == 0),
            EQ: lambda: int((a - b) % P == 0), IS_NEG: lambda: (a % P) & 1, SQR_N: lambda: pow(a, 1 << b, P)}[op]()


EXACT_OPS = (CANON, IS_ZERO, EQ, IS_NEG)  # results that are canonical values or 0 / 1: equal to the truth, not just congruent


def _split_fold(a, b):
    """The first fold as fe_mul_asm / fe_sqr_asm compute it: the product is held as two interleaved column sums, E (products a_i b_j
    with i + j even) and O (i + j odd), and each half folds on its own, so the carry of E_lo + O_lo never reaches the high half:
    v1' = E_lo + O_lo + 38 (E_hi + O_hi) = v1 + c (2^256 - 38), c that carry.  (The result bits are still the model's: fold2(v) and
    fold2(v + 2p) differ only for v < 38, where ab < 38 and c = 0.)"""
    la, lb = [(a >> (32 * i)) & M32 for i in range(8)], [(b >> (32 * i)) & M32 for i in range(8)]
    E = sum(la[i] * lb[j] << (32 * (i + j)) for i in range(8) for j in range(8) if (i + j) % 2 == 0)
    O = sum(la[i] * lb[j] << (32 * (i + j)) for i in range(8) for j in range(8) if (i + j) % 2 == 1)
    return E % T + O % T + 38 * ((E >> 256) + (O >> 256))


def path(op, a, b):
    """'wrap' (the ripple and its second wrap), 'ripple' (the ripple alone) or 'plain': the path of the generated PTX for one input."""
    if op in (MUL, SQR, ADD):
        v1 = a + b if op == ADD else _split_fold(a, a if op == SQR else b)
        lo, top = v1 % T, v1 >> 256
        return "wrap" if lo + 38 * top >= T else "ripple" if (lo & M32) + 38 * top > M32 else "plain"
    d = -a if op == NEG else a - b
    if d >= 0:
        return "plain"
    return "wrap" if d + T - 38 < 0 else "ripple" if (d % T) & M32 < 38 else "plain"


# ---------------------------------------------------------------------------------------------------- input classes
def _sqrt_mod_2p(s):
    """a with a^2 = s (mod 2p), or None when s is not a square mod p (p = 5 mod 8: one exponentiation, then sqrt(-1))."""
    if s % P == 0 or pow(s, (P - 1) // 2, P) != 1:
        return None
    x = pow(s, (P + 3) // 8, P)
    if x * x % P != s % P:
        x = x * pow(2, (P - 1) // 4, P) % P
    return x + P if x % 2 != s % 2 else x  # a^2 = s mod 2 as well


def _noncanonical(rnd):
    """Operands that are not canonical: [p, 2^256), 2p (= 0), 2^255 + k, and limbs of 0xFFFFFFFF."""
    vals = [P + k for k in (0, 1, 2, 18, 19, 37)] + [M - 1, M, M + 1, T - 1, T - 2, T - 19, T - 37, T - 39]
    vals += [(1 << 255) + k for k in (0, 1, 18, 19, 20, 37, 38)]
    for _ in range(16):   # 0xFFFFFFFF in a random set of limbs, random words elsewhere
        v = rnd.getrandbits(256)
        for k in range(8):
            if rnd.random() < 0.6:
                v |= M32 << (32 * k)
        vals.append(v)
    vals += [sum(M32 << (32 * k) for k in range(1, 8)) | rnd.getrandbits(32) for _ in range(4)]
    vals += [rnd.randrange(P, T) for _ in range(8)]
    return vals


def fe_classes():
    """{class name: (op, [(a, b)], path the model must find, minimum count of that path)}."""
    rnd = random.Random(20261017)
    C = {}
    pairs = []
    while len(pairs) < 160:   # b = s a^-1 mod 2p, s in [39, 75]: two folds leave s - 38 + 2^256, the last +38 wraps to s
        a = rnd.getrandbits(256) | 1
        if a % P:
            pairs.append((a, rnd.randrange(39, 76) * pow(a, -1, M) % M))
    C["mul_wrap"] = (MUL, pairs, "wrap", 120)
    pairs = []
    while len(pairs) < 160:   # a b = s (mod 2p) with s = hi 2^32 + (< 38): the fold's +38 q carries out of limb 0 and stops in limb 1
        a = rnd.getrandbits(256) | 1
        if a % P:
            pairs.append((a, ((rnd.getrandbits(220) << 32) | rnd.randrange(38)) * pow(a, -1, M) % M))
    C["mul_ripple"] = (MUL, pairs, "ripple", 140)
    sq = []
    for s in range(39, 400):
        x = _sqrt_mod_2p(s)
        if x is not None:
            sq += [(x, 0), ((P - x) + (P if (P - x) % 2 != s % 2 else 0), 0)]
    C["sqr_wrap"] = (SQR, sq, "wrap", 100)
    sq = []
    while len(sq) < 160:
        x = _sqrt_mod_2p((rnd.getrandbits(220) << 32) | rnd.randrange(38))
        if x is not None:
            sq.append((x, 0))
    C["sqr_ripple"] = (SQR, sq, "ripple", 140)
    pairs = []
    for _ in range(120):      # a + b = 2^256 + t, t's low limb within 38 of 2^32
        t = (rnd.getrandbits(200) << 32) | (M32 - rnd.randrange(38))
        a = rnd.randrange(t + 1, T)
        pairs.append((a, T + t - a))
    C["add_ripple"] = (ADD, pairs, "ripple", 120)
    C["add_wrap"] = (ADD, [(T - 1 - rnd.randrange(19), T - 1 - rnd.randrange(19)) for _ in range(120)], "wrap", 120)
    pairs = []
    for _ in range(120):      # a - b = t - 2^256, t's low limb below 38
        t = (rnd.getrandbits(200) << 32) | rnd.randrange(38)
        a = rnd.randrange(t)
        pairs.append((a, a - t + T))
    C["sub_ripple"] = (SUB, pairs, "ripple", 120)
    pairs = []
    for _ in range(120):      # a - b + 2^256 - 38 < 0
        a = rnd.randrange(37)
        pairs.append((a, T - 1 - rnd.randrange(37 - a)))
    C["sub_wrap"] = (SUB, pairs, "wrap", 120)
    C["neg_wrap"] = (NEG, [(T - 1 - k, 0) for k in range(37)], "wrap", 37)   # 0 - a with a > 2^256 - 38
    nc = _noncanonical(rnd)
    rv = [rnd.getrandbits(256) for _ in range(64)]
    for op in (MUL, ADD, SUB):
        C["noncanonical_%d" % op] = (op, [(x, y) for x in nc for y in nc[::3]], None, 0)
        C["random_%d" % op] = (op, list(zip(rv, rv[1:] + rv[:1])) + [(x, y) for x in nc[:8] for y in rv[:8]], None, 0)
    for op in (SQR, NEG, CANON, IS_NEG, IS_ZERO):
        C["noncanonical_%d" % op] = (op, [(x, 0) for x in nc + rv], None, 0)
    # canonicalisation and the predicates at [p, 2^255 + 19) and [2^255, 2^256), and equality across representations
    edge = [P + k for k in range(38)] + [(1 << 255) + k for k in range(40)] + [T - 1 - k for k in range(40)] + [rnd.randrange(1 << 255, T) for _ in range(40)]
    for op in (CANON, IS_ZERO, IS_NEG):
        C["edge_%d" % op] = (op, [(x, 0) for x in edge], None, 0)
    eq = [(x, x % P) for x in edge] + [(x, x % P + 1) for x in edge] + [(x % P, x) for x in edge] + [(0, M), (M, 0), (P, M), (0, P), (1, P + 1), (T - 1, 37)]
    C["edge_eq"] = (EQ, eq, None, 0)
    # the exponentiation chains on 0, p, 2p, the edges and what the wrap classes produce
    wraps = [m_mul(a, b) for a, b in C["mul_wrap"][1][:12]] + [m_sqr(a) for a, _ in C["sqr_wrap"][1][:12]]
    chain = [0, 1, P, M, P + 1, T - 1, T - 38, 1 << 255] + wraps + [a for a, _ in C["sqr_wrap"][1][:8]] + rv[:8]
    C["chain_invert"] = (INVERT, [(x, 0) for x in chain], None, 0)
    C["chain_pow_p58"] = (POW_P58, [(x, 0) for x in chain], None, 0)
    C["sqr_n"] = (SQR_N, [(a, n) for a, _ in C["sqr_wrap"][1][:40] for n in (1, 2, 7)] + [(x, 5) for x in nc[:20]], None, 0)
    return C


def test_model_classes_take_their_paths():
    """The crafted classes reach the paths they are built for (checked on the model, so it also guards the class builders), and the
    models agree with Python integers mod p."""
    for name, (op, pairs, want, least) in fe_classes().items():
        got = 0
        for a, b in pairs:
            r = model(op, a, b)
            assert 0 <= r < T and (r == truth(op, a, b) if op in EXACT_OPS else r % P == truth(op, a, b)), (name, hex(a), hex(b))
            if want:
                got += path(op, a, b) == want
        assert got >= least, (name, got, least)


# ---------------------------------------------------------------------------------------------------- the generator
def _gen_module():
    spec = importlib.util.spec_from_file_location("gen_fe_asm", os.path.join(ROOT, "tools", "gen_fe_asm.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_committed_fe_asm_is_the_generated_one():
    """render() runs every simulation check (each asserts how often the ripple and the second wrap ran) and returns the header: a hand
    edit of fe_asm.cuh, which the host emulation never compiles, fails here."""
    with open(os.path.join(ROOT, "hotstuff_b200", "csrc", "fe_asm.cuh")) as f:
        assert f.read() == _gen_module().render(), "fe_asm.cuh differs from what tools/gen_fe_asm.py emits: rerun the generator"


def test_generator_simulation_takes_the_rare_paths():
    """The generator's own PTX simulator on the crafted classes: the sequences it emits take the ripple and the second wrap there, and
    give the model's bits."""
    g = _gen_module()
    progs = {MUL: g.gen_mul(), SQR: g.gen_sqr(split=True), ADD: g.gen_add(), SUB: g.gen_sub()}
    tags = {MUL: "red", SQR: "red", ADD: "add", SUB: "sub"}
    for name, (op, pairs, want, least) in fe_classes().items():
        if op not in progs:
            continue
        taken = 0
        for a, b in pairs:
            env = {"a%d" % i: (a >> (32 * i)) & M32 for i in range(8)}
            if op != SQR:
                env.update({"b%d" % i: (b >> (32 * i)) & M32 for i in range(8)})
            trace = set()
            out = progs[op].run(env, trace)
            r = sum(out["r%d" % i] << (32 * i) for i in range(8))
            assert r == model(op, a, b), (name, hex(a), hex(b))
            p = ("wrap" if out.get("w_" + tags[op], 0) else "ripple") if "L_" + tags[op] in trace else "plain"
            assert p == path(op, a, b), (name, hex(a), hex(b), p)
            taken += p == want
        assert taken >= least, (name, taken)   # least is 0 for the classes without a target path


# ---------------------------------------------------------------------------------------------------- host emulation
@pytest.fixture(scope="module")
def arith_emu(tmp_path_factory):
    """tests/hostemu/arith_emu.cpp: the harness's field op table (tests/cuda/arith_ops.cuh) built by g++ with the portable C."""
    lib = str(tmp_path_factory.mktemp("arith_emu") / "libarith_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "arith_emu.cpp")])
    lib = ctypes.CDLL(lib)
    lib.emu_arith_fe_op.restype = None
    lib.emu_arith_fe_op.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return lib


def _fe_call(fn, op, pairs):
    """fn(op, a, b, out, n) over host arrays of 8-word elements -> the n results as integers."""
    a, b = _words([p[0] for p in pairs], 8), _words([p[1] for p in pairs], 8)
    out = np.zeros_like(a)
    rc = fn(op, a.ctypes.data, b.ctypes.data, out.ctypes.data, len(pairs))
    assert not rc, "CUDA error %d" % rc
    return [sum(int(w) << (32 * i) for i, w in enumerate(row)) for row in out]


def test_hostemu_equals_the_models_bit_for_bit(arith_emu, hostemu):
    """The premise that host-emulation results carry over to the device, at the level of bits: the portable C of every primitive gives
    exactly the model's representation on every class, through the harness's op table and (ops 0..7) through emu_fe_op."""
    o = ctypes.create_string_buffer(32)
    for name, (op, pairs, _, _) in fe_classes().items():
        for (a, b), r in zip(pairs, _fe_call(arith_emu.emu_arith_fe_op, op, pairs)):
            assert r == model(op, a, b), (name, op, hex(a), hex(b))
            if op <= NEG:
                hostemu.emu_fe_op(op, a.to_bytes(32, "little"), b.to_bytes(32, "little"), o)
                assert int.from_bytes(o.raw, "little") == r, (name, op, hex(a), hex(b))


def _scalar_edges():
    rng = random.Random(7)
    xs = [rng.getrandbits(512) for _ in range(300)]
    xs += [0, L_ORDER - 1, L_ORDER, L_ORDER + 1, 2**512 - 1, (2**512 // L_ORDER) * L_ORDER, (2**512 // L_ORDER) * L_ORDER - 1, L_ORDER << 259]
    xs += [2**512 - 1 - rng.getrandbits(160) for _ in range(50)] + [L_ORDER * rng.getrandbits(259) + d for d in (-1, 0, 1) for _ in range(20)]
    canon = [0, 1, L_ORDER - 1, L_ORDER, L_ORDER + 1, 2**252, 2**253, 2**256 - 1] + [L_ORDER + d for d in range(-40, 40)] + [rng.getrandbits(256) for _ in range(50)]
    return [x % 2**512 for x in xs], canon


def ndigits(w):
    r = 253 % w
    return (253 + w - 1) // w + (1 if r in (0, w - 1) else 0)


def signed_digits(s, w):
    """sc_digits_rt's recoding: digit i = bits [w i, w i + w) of s + sum_i 2^(w - 1 + w i), minus 2^(w - 1)."""
    n = ndigits(w)
    u = s + sum(1 << (w - 1 + w * i) for i in range(n))
    return [((u >> (w * i)) & ((1 << w) - 1)) - (1 << (w - 1)) for i in range(n)]


def digit_scalars(w):
    """Scalars below 2^253 whose non-top digits are all -2^(w-1) (each gathers its window's last entry), all 0 (the identity
    entry), or alternate between the two, plus the recoding edges and random scalars below l."""
    n, half = ndigits(w), 1 << (w - 1)
    top = 1 << (w * (n - 1))
    all_min = top - sum(half << (w * i) for i in range(n - 1))
    alt = top - sum(half << (w * i) for i in range(0, n - 1, 2))
    rng = random.Random(w)
    s = [all_min, alt, 0, top, 2 * top, top - 1, 1, L_ORDER - 1, 2**253 - 1, 2**252, int("7f" * 31, 16), int("80" * 31, 16)]
    s += [rng.randrange(L_ORDER) for _ in range(40)]
    s = [x for x in s if x < 2**253]
    assert signed_digits(all_min, w)[:-1] == [-half] * (n - 1) and signed_digits(top, w)[:-1] == [0] * (n - 1)
    assert signed_digits(alt, w)[:-1:2] == [-half] * ((n - 1 + 1) // 2) and set(signed_digits(alt, w)[1:-1:2]) <= {0}
    return s


def test_hostemu_scalar_edges(hostemu):
    xs, canon = _scalar_edges()
    for x in xs:
        o = ctypes.create_string_buffer(32)
        hostemu.emu_sc_reduce512(x.to_bytes(64, "little"), o)
        assert int.from_bytes(o.raw, "little") == x % L_ORDER, hex(x)
    for s in canon:
        assert hostemu.emu_sc_is_canonical(s.to_bytes(32, "little")) == int(s < L_ORDER), hex(s)
    for w in range(8, 27):
        for s in digit_scalars(w):
            out = (ctypes.c_int * 80)()
            n = hostemu.emu_sc_digits(w, 0, s.to_bytes(32, "little"), out)
            d = list(out)[:n]
            assert d == signed_digits(s, w) and sum(x << (w * i) for i, x in enumerate(d)) == s, (w, hex(s))


# ---------------------------------------------------------------------------------------------------- the device harness
@pytest.fixture(scope="module")
def harness_path(tmp_path_factory):
    """tests/cuda/arith_harness.cu built for sm_90a into a temporary directory (never into the product library)."""
    from hotstuff_b200 import build
    out = str(tmp_path_factory.mktemp("arith") / "libarith_harness.so")
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
    subprocess.check_call([nvcc] + build.NVCC_FLAGS + ["-o", out, HARNESS], cwd=build.ROOT)
    return out


def test_harness_compiles_for_sm90a(harness_path):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else "cuobjdump", "--list-elf",
                          harness_path], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in out, out


@pytest.fixture(scope="module")
def harness(harness_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = ctypes.CDLL(harness_path)
    lib.arith_fe_op.restype = ctypes.c_int
    lib.arith_fe_op.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.arith_sc_op.restype = ctypes.c_int
    lib.arith_sc_op.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return lib


def _words(vals, n_words):
    return np.array([[(v >> (32 * i)) & M32 for i in range(n_words)] for v in vals], dtype=np.uint32)


@pytest.mark.gpu
def test_device_field_ops_equal_model_emulation_and_integers(harness, arith_emu):
    """Every class through the PTX primitives: the device result is the model's bits, the host emulation's bits, and right mod p.  A
    change to one of the fold constants of fe_asm.cuh fails the wrap classes here."""
    bad = {}  # class -> (mismatches, first mismatch): every failing class is named, not only the first
    for name, (op, pairs, want, least) in fe_classes().items():
        dev = _fe_call(harness.arith_fe_op, op, pairs)
        for (a, b), r, e in zip(pairs, dev, _fe_call(arith_emu.emu_arith_fe_op, op, pairs)):
            ok = r == model(op, a, b) and r == e
            ok = ok and ((r == truth(op, a, b)) if op in EXACT_OPS else (r % P == truth(op, a, b)))
            if not ok:
                n, first = bad.get(name, (0, (hex(a), hex(b), hex(r))))
                bad[name] = (n + 1, first)
        if want:
            assert sum(path(op, a, b) == want for a, b in pairs) >= least, name
    assert not bad, "; ".join("%s: %d wrong, first (a, b, device) = %s" % (k, n, first) for k, (n, first) in sorted(bad.items()))


def _device_sc(lib, op, w, vals, n_words):
    x = np.zeros((len(vals), 16), np.uint32)
    x[:, :n_words] = _words(vals, n_words)
    out = np.zeros((len(vals), 64), np.int32)
    rc = lib.arith_sc_op(op, w, x.ctypes.data, out.ctypes.data, len(vals))
    assert rc == 0, "CUDA error %d" % rc
    return out


@pytest.mark.gpu
def test_device_scalar_ops_equal_emulation_and_integers(harness, hostemu):
    xs, canon = _scalar_edges()
    out = _device_sc(harness, 0, 0, xs, 16)
    for x, row in zip(xs, out):
        r = sum((int(v) & M32) << (32 * i) for i, v in enumerate(row[:8]))
        o = ctypes.create_string_buffer(32)
        hostemu.emu_sc_reduce512(x.to_bytes(64, "little"), o)
        assert r == x % L_ORDER == int.from_bytes(o.raw, "little"), hex(x)
    out = _device_sc(harness, 1, 0, canon, 8)
    for s, row in zip(canon, out):
        assert int(row[0]) == int(s < L_ORDER) == hostemu.emu_sc_is_canonical(s.to_bytes(32, "little")), hex(s)
    for w in range(8, 27):
        vals = digit_scalars(w)
        out = _device_sc(harness, 2, w, vals, 8)
        n = ndigits(w)
        for s, row in zip(vals, out):
            emu = (ctypes.c_int * 80)()
            assert hostemu.emu_sc_digits(w, 0, s.to_bytes(32, "little"), emu) == n
            assert [int(v) for v in row[:n]] == signed_digits(s, w) == list(emu)[:n], (w, hex(s))


# ---------------------------------------------------------------------------------------------------- edge-digit signatures
def _edge():
    with open(EDGE) as f:
        return json.load(f)


def _record_scalars(r):
    sig, pk, msg = bytes.fromhex(r["sig"]), bytes.fromhex(r["pk"]), bytes.fromhex(r["msg"])
    k = int.from_bytes(hashlib.sha512(sig[:32] + pk + msg).digest(), "little") % L_ORDER
    return {"k": k, "S": int.from_bytes(sig[32:], "little")}


def test_edge_digit_fixture_makes_every_claim(oracle):
    """Each claim of tests/golden/edge_digits.json recomputed from the record's bytes (k = SHA-512(R || A || M) mod l, S from the
    signature), every claim the GPU test relies on present, and every record a valid signature by its seed."""
    doc = _edge()
    recs = doc["records"]
    assert doc["key_widths"] == list(range(8, 18)) and doc["base_widths"] == [16, 20, 24]
    made = set()
    for r in recs:
        sc = _record_scalars(r)
        assert sc["S"] < L_ORDER
        for c in r["covers"]:
            name, w, kind, i = re.fullmatch(r"([kS])(\d+):(min|zero)@(\d+)", c).groups()
            w, i = int(w), int(i)
            d = signed_digits(sc[name], w)
            assert sum(x << (w * j) for j, x in enumerate(d)) == sc[name]
            assert i < len(d) - 1, c                                        # a non-top digit
            assert d[i] == (-(1 << (w - 1)) if kind == "min" else 0), (c, d[i])
            if name == "k" and kind == "zero":
                assert i == 0, c                                            # k's window 0: the identity is the comb's first accumulator
            made.add("%s%d:%s" % (name, w, kind))
    want = {"k%d:%s" % (w, c) for w in range(8, 18) for c in ("min", "zero")} | {"S%d:%s" % (w, c) for w in (16, 20, 24) for c in ("min", "zero")}
    assert want <= made, sorted(want - made)
    assert len({r["pk"] for r in recs}) <= 4                                # small per-key tables
    seeds = np.array([list(bytes.fromhex(r["seed"])) for r in recs], np.uint8)
    assert [bytes(p).hex() for p in oracle.keygen_batch(seeds)] == [r["pk"] for r in recs]
    recs128, expect = _edge_records()
    assert (oracle.verify_rec128(recs128) == (expect & 1).astype(bool)).all()
    assert (oracle.verify_rec128(recs128, mode=1) == (expect >> 1).astype(bool)).all()


def _edge_records():
    """The fixture's records, each followed by a copy with bit 0 of its message flipped; expect bytes 3 (strict and batch-eq) and 0."""
    rows, expect = [], []
    for r in _edge()["records"]:
        rec = bytes.fromhex(r["sig"] + r["pk"] + r["msg"])
        bad = bytearray(rec)
        bad[96] ^= 1
        rows += [list(rec), list(bad)]
        expect += [3, 0]
    return np.array(rows, np.uint8), np.array(expect, np.uint8)


def _edge_on(eng, oracle, key_bits=range(8, 18)):
    recs, expect = _edge_records()
    for kb in key_bits:
        failed = eng.self_test(recs=recs, expect=expect, key_bits=kb)
        assert failed == 0, (kb, hex(failed), eng.last_error)
    want = oracle.verify_rec128(recs)
    assert (eng.verify_rec128(recs) == want).all()
    pks = sorted({bytes(r[64:96]) for r in recs})
    vidx = np.array([pks.index(bytes(r[64:96])) for r in recs], np.uint32)
    try:
        assert eng.committee_register(np.array([list(p) for p in pks], np.uint8)).all()
        assert (eng.verify_committee(vidx, recs[:, :64], recs[:, 96:], msg_idx=np.arange(len(recs), dtype=np.uint32)) == want).all()
        assert (eng.verify_rec128(recs) == want).all()                   # through the key lookup
    finally:
        eng.committee_register(np.zeros((0, 32), np.uint8))


@pytest.mark.gpu
def test_edge_digit_signatures_on_every_verify_path_at_the_default_geometry(engine, oracle):
    """The fixture's records and their flipped copies through every verify path (HS_SELFTEST_VERIFY_PATHS) at every key width 8..17 on
    the default 24-bit base table, then verify_rec128 and verify_committee against the oracle.  Base width 26 (a 32 GB table) is left out
    on purpose: the GPUs these tests run on are shared."""
    assert engine.window_bits[1] == 24, engine.window_bits
    _edge_on(engine, oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("base_window", [16, 20])
def test_edge_digit_signatures_on_every_verify_path_at_narrow_base_windows(oracle, base_window):
    """The same at base widths 16 and 20 (about 50 MB and 650 MB of base table), each on a context of its own, closed at the end."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import Engine, build
    build.build_engine()
    eng = Engine(0, base_window=base_window)
    try:
        assert eng.window_bits[1] == base_window
        _edge_on(eng, oracle)
    finally:
        eng.close()
