#!/usr/bin/env python3
"""EXPERIMENT (not kept: slower per dependent squaring than the saturated multiplier, tools/microbench/latency.cu).  Generate tools/experiments/fe10.cuh: GF(2^255-19) multiply / square on TEN unsaturated limbs (26/25 bits alternating) — the
LATENCY representation used by the one-warp-per-signature path (k_verify_small).

Why a second representation: the saturated 8 x 32 multiplier (fe_asm.cuh) is the throughput choice (72 wide multiplies instead of
100) but every one of its instructions hangs on the carry flag of the previous one, so ONE dependent fe_sqr takes hundreds of cycles
(tools/microbench/latency.cu) and the 252-squaring square-root chain of a point decompression dominates the latency of a lone warp.  With 25.5-bit limbs the 100 (55) partial products are independent 64-bit multiply-accumulates (no carries until one
short interleaved pass at the end), which a single warp can issue back to back.

Every formula is generated from the rule  f_i g_j -> h_((i+j) mod 10), x19 if i+j >= 10, x2 if i and j are both odd,
and the generator checks the emitted formulas against Python big integers before writing the header.
"""
import os
import random

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
P = 2**255 - 19
OFF = [0, 26, 51, 77, 102, 128, 153, 179, 204, 230]
BITS = [26, 25, 26, 25, 26, 25, 26, 25, 26, 25]


def terms_mul():
    h = [[] for _ in range(10)]
    for i in range(10):
        for j in range(10):
            k = (i + j) % 10
            c = (19 if i + j >= 10 else 1) * (2 if (i & 1) and (j & 1) else 1)
            h[k].append((i, j, c))
    return h


def terms_sqr():
    h = [[] for _ in range(10)]
    for i in range(10):
        for j in range(i, 10):
            k = (i + j) % 10
            c = (19 if i + j >= 10 else 1) * (2 if (i & 1) and (j & 1) else 1) * (1 if i == j else 2)
            h[k].append((i, j, c))
    return h


def to10(x):
    x %= P
    return [(x >> OFF[i]) & ((1 << BITS[i]) - 1) for i in range(10)]


def from10(v):
    return sum(int(x) << OFF[i] for i, x in enumerate(v)) % P


CARRY_ORDER = [0, 4, 1, 5, 2, 6, 3, 7, 4, 8, 9, 0]   # ref10's interleaved order: two chains in flight


def carry(h):
    h = list(h)
    for i in CARRY_ORDER:
        c = h[i] >> BITS[i]
        h[i] &= (1 << BITS[i]) - 1
        if i == 9:
            h[0] += 19 * c
        else:
            h[i + 1] += c
    return h


def simulate(terms, f, g):
    h = [sum(c * f[i] * g[j] for i, j, c in t) for t in terms]
    assert max(h) < 2**64, "64-bit accumulator overflow"
    return carry(h)


def selftest():
    rnd = random.Random(10)
    tm, ts = terms_mul(), terms_sqr()
    worst = [(1 << 26) + 600] * 10        # above anything the carry pass leaves behind (limb 0/1 excess is < 2^10)
    assert all(sum(c * worst[i] * worst[j] for i, j, c in t) < 2**64 for t in tm)
    cases = [(to10(rnd.randrange(P)), to10(rnd.randrange(P))) for _ in range(300)] + [(worst, worst), (to10(P - 1), to10(P - 1)), (to10(0), to10(5))]
    for f, g in cases:
        r = simulate(tm, f, g)
        assert from10(r) == from10(f) * from10(g) % P
        assert all(x < (1 << BITS[i]) + 600 for i, x in enumerate(r)), r
        r = simulate(ts, f, f)
        assert from10(r) == from10(f) ** 2 % P


def emit(terms, name, two_ops):
    L = []
    args = "fe10 &h, const fe10 &f, const fe10 &g" if two_ops else "fe10 &h, const fe10 &f"
    L.append("HS_HD void %s(%s) {" % (name, args))
    g = "g" if two_ops else "f"
    # pre-scaled operands: products stay 32 x 32 -> 64 (IMAD.WIDE): the small constant goes onto one 32-bit factor
    scaled = {}
    for t in terms:
        for i, j, c in t:
            if c != 1:
                scaled[(j, c)] = True
    for (j, c) in sorted(scaled):
        # g_j * c must fit in 32 bits: limbs < 2^26 + 600, c <= 76  ->  < 2^32.3 for c = 76: split 76 = 2 * 38 below
        pass
    L.append("  const uint32_t *F = f.v, *G = %s.v;" % g)
    L.append("  uint64_t t[10];")
    for k, t in enumerate(terms):
        parts = []
        for i, j, c in t:
            if c == 1:
                parts.append("(uint64_t)F[%d] * G[%d]" % (i, j))
            elif c <= 38:
                parts.append("(uint64_t)F[%d] * (G[%d] * %du)" % (i, j, c))      # G * 38 < 2^32 for G < 2^26.7
            else:                                                                 # 76 = 2 * 38: put the 2 on the other factor
                parts.append("(uint64_t)(F[%d] * 2u) * (G[%d] * %du)" % (i, j, c // 2))
        L.append("  t[%d] = %s;" % (k, " + ".join(parts)))
    L.append("  fe10_carry(h, t);")
    L.append("}")
    return L


STATIC = r'''
// ---- conversions (8 x 32 saturated, any representative below 2^256  <->  ten limbs)
HS_HD void fe10_from_fe(fe10 &r, const fe &a) {
  // fold bit 255 (2^255 = 19): 255 bits + at most 19 remain; a second bit 255 (value within 19 of 2^255) just widens limb 9 by one bit
  uint32_t w[8];
  uint64_t acc = (uint64_t)(a.v[7] >> 31) * 19u;
  for (int i = 0; i < 8; i++) {
    acc += (i == 7) ? (a.v[7] & 0x7fffffffu) : a.v[i];
    w[i] = (uint32_t)acc;
    acc >>= 32;
  }
  const int off[10] = {0, 26, 51, 77, 102, 128, 153, 179, 204, 230};
  for (int i = 0; i < 10; i++) {
    const int word = off[i] >> 5, sh = off[i] & 31;
    uint64_t two = (uint64_t)w[word] | ((word < 7) ? ((uint64_t)w[word + 1] << 32) : 0);
    uint32_t v = (uint32_t)(two >> sh);
    r.v[i] = (i == 9) ? v : (v & ((i & 1) ? 0x1ffffffu : 0x3ffffffu));
  }
}
HS_HD void fe10_to_fe(fe &r, const fe10 &a) {
  const int off[10] = {0, 26, 51, 77, 102, 128, 153, 179, 204, 230};
  uint64_t t[9];
  for (int i = 0; i < 9; i++) t[i] = 0;
  for (int i = 0; i < 10; i++) {
    const int word = off[i] >> 5, sh = off[i] & 31;
    const uint64_t v = (uint64_t)a.v[i] << sh;  // limbs < 2^27, sh <= 31
    t[word] += v & 0xffffffffu;
    t[word + 1] += v >> 32;
  }
  uint64_t carry = 0;
  for (int i = 0; i < 8; i++) {
    t[i] += carry;
    r.v[i] = (uint32_t)t[i];
    carry = t[i] >> 32;
  }
  // limb 9 < 2^26 at bit 230: the total stays below 2^256 (t[8] + carry == 0); fold defensively all the same
  uint64_t top = (t[8] + carry) * 38u;
  for (int i = 0; i < 8 && top; i++) {
    top += r.v[i];
    r.v[i] = (uint32_t)top;
    top >>= 32;
  }
}
HS_HD void fe10_sqr_n(fe10 &r, const fe10 &a, int n) {
  fe10_sqr(r, a);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 1; i < n; i++) fe10_sqr(r, r);
}
// z^(2^250-1) and z^11: the same addition chain as fe_pow2_250_1 (fe.cuh)
HS_HD void fe10_pow2_250_1(fe10 &out, fe10 &z11, const fe10 &z) {
  fe10 z2, z9, t, a, b, c;
  fe10_sqr(z2, z);
  fe10_sqr_n(t, z2, 2);
  fe10_mul(z9, t, z);
  fe10_mul(z11, z9, z2);
  fe10_sqr(t, z11);
  fe10_mul(a, t, z9);
  fe10_sqr_n(t, a, 5);
  fe10_mul(b, t, a);
  fe10_sqr_n(t, b, 10);
  fe10_mul(c, t, b);
  fe10_sqr_n(t, c, 20);
  fe10_mul(t, t, c);
  fe10_sqr_n(t, t, 10);
  fe10_mul(b, t, b);
  fe10_sqr_n(t, b, 50);
  fe10_mul(c, t, b);
  fe10_sqr_n(t, c, 100);
  fe10_mul(t, t, c);
  fe10_sqr_n(t, t, 50);
  fe10_mul(out, t, b);
}
// latency variants of fe_invert / fe_pow_p58: convert, run the chain on ten limbs, convert back
HS_HD void fe_invert_lat(fe &r, const fe &z) {
  fe10 x, t, z11;
  fe10_from_fe(x, z);
  fe10_pow2_250_1(t, z11, x);
  fe10_sqr_n(t, t, 5);
  fe10_mul(t, t, z11);
  fe10_to_fe(r, t);
}
HS_HD void fe_pow_p58_lat(fe &r, const fe &z) {
  fe10 x, t, z11;
  fe10_from_fe(x, z);
  fe10_pow2_250_1(t, z11, x);
  fe10_sqr_n(t, t, 2);
  fe10_mul(t, t, x);
  fe10_to_fe(r, t);
}
'''


def main():
    selftest()
    out = []
    out.append("// GENERATED by tools/gen_fe10.py — do not edit.  GF(2^255-19) on ten unsaturated limbs (26/25 bits): the latency representation.")
    out.append("// value = sum v[i] * 2^ceil(25.5 i); limbs stay below 2^26 + 600 between operations; formulas checked against big integers.")
    out.append("#pragma once")
    out.append("#include <cstdint>")
    out.append('#include "../../hotstuff_b200/csrc/fe.cuh"')
    out.append("")
    out.append("struct fe10 {")
    out.append("  uint32_t v[10];")
    out.append("};")
    out.append("// one interleaved carry pass (two chains in flight: 0->1->2->3->4 and 4->5->...->9->0->1), 64-bit columns -> limbs")
    out.append("HS_HD void fe10_carry(fe10 &h, uint64_t (&t)[10]) {")
    for i in CARRY_ORDER:
        if i == 9:
            out.append("  t[0] += 19u * (t[9] >> 25); t[9] &= 0x1ffffffu;")
        else:
            out.append("  t[%d] += t[%d] >> %d; t[%d] &= 0x%xu;" % (i + 1, i, BITS[i], i, (1 << BITS[i]) - 1))
    out.append("  for (int i = 0; i < 10; i++) h.v[i] = (uint32_t)t[i];")
    out.append("}")
    out += emit(terms_mul(), "fe10_mul", True)
    out += emit(terms_sqr(), "fe10_sqr", False)
    out.append(STATIC)
    with open(os.path.join(ROOT, "tools", "experiments", "fe10.cuh"), "w") as f:
        f.write("\n".join(out) + "\n")
    print("wrote fe10.cuh")


if __name__ == "__main__":
    main()
