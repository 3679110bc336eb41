#!/usr/bin/env python3
"""Generate the inline-PTX field multiplication / squaring for GF(2^255-19) on sm_90a.

Representation: 8 saturated 32-bit limbs, value in [0, 2^256), congruent mod p = 2^255-19
(2^256 = 38 mod p).  The schoolbook products are laid out as `mad.lo.cc.u32` / `madc.hi.cc.u32`
pairs on two interleaved accumulator arrays (even / odd columns) so that ptxas fuses every pair into a
single `IMAD.WIDE.U32.X Rd, Pc, Ra, Rb, Rd, Pc` (64-bit multiply-accumulate with carry-in/out), i.e. one
SASS instruction per 32x32 partial product and no separate carry handling (issue rates: tools/microbench/pipes.cu).

The generator builds an abstract instruction list, *simulates it in Python against big-integer
arithmetic* (random + all-ones + edge inputs) and only then emits PTX, so a lost carry cannot reach the GPU.

Output: hotstuff_b200/csrc/fe_asm.cuh
"""
import os
import random

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = (1 << 32) - 1
P = 2**255 - 19


class Prog:
    def __init__(self):
        self.ops = []          # (mnemonic, dst, [srcs])  srcs are reg names or ints
        self.tmp = set()

    def emit(self, op, dst, *srcs):
        self.ops.append((op, dst, list(srcs)))

    # ---- simulation -----------------------------------------------------
    def run(self, env, trace=None):
        cc = 0
        env = dict(env)

        def val(x):
            return x if isinstance(x, int) else env[x]

        labels = {dst: i for i, (op, dst, _) in enumerate(self.ops) if op == "label"}
        pc = 0
        while pc < len(self.ops):
            op, dst, srcs = self.ops[pc]
            pc += 1
            if op == "label":
                continue
            if op == "setp.lt.u32":
                env[dst] = 1 if val(srcs[0]) < val(srcs[1]) else 0
                continue
            if op == "bra_if_not":        # dst = predicate, srcs[0] = label: the common (fall-through-skipping) path
                if not env[dst]:
                    pc = labels[srcs[0]]
                elif trace is not None:
                    trace.add(srcs[0])
                continue
            s = [val(x) for x in srcs]
            base = op.replace(".u32", "")
            if base in ("mul.lo", "mul.hi"):
                pr = s[0] * s[1]
                env[dst] = (pr & M32) if base == "mul.lo" else (pr >> 32)
                continue
            if base == "shf.l":
                env[dst] = ((s[1] << s[2]) | (s[0] >> (32 - s[2]))) & M32
                continue
            if base == "and":
                env[dst] = s[0] & s[1]
                continue
            parts = base.split(".")
            name = parts[0]
            cin = name.endswith("c") and name in ("madc", "addc", "subc")
            cout = parts[-1] == "cc"
            if name in ("mad", "madc"):
                pr = s[0] * s[1]
                pr = (pr & M32) if parts[1] == "lo" else (pr >> 32)
                t = pr + s[2] + (cc if cin else 0)
            elif name in ("add", "addc"):
                t = s[0] + s[1] + (cc if cin else 0)
            elif name in ("sub", "subc"):
                t = s[0] - s[1] - (cc if cin else 0)
            else:
                raise ValueError(op)
            env[dst] = t & M32
            if cout:
                cc = 1 if (t < 0 or t > M32) else 0
            # (PTX leaves CC unchanged when .cc is absent)
        return env

    # ---- PTX text -------------------------------------------------------
    def ptx(self, operand):
        """operand: map reg name -> asm operand string ('%3') for inputs/outputs; others become .reg temps"""
        temps = []
        seen = set()
        for op, dst, srcs in self.ops:
            if op == "label":
                continue
            for r in [dst] + [x for x in srcs if not isinstance(x, int) and not str(x).startswith("L_")]:
                if r not in operand and r not in seen:
                    seen.add(r)
                    temps.append(r)
        preds = [t for t in temps if t.startswith("p_")]
        temps = [t for t in temps if not t.startswith("p_") and not t.startswith("L_")]
        lines = ["{"]
        for i in range(0, len(temps), 12):
            lines.append(".reg .u32 " + ", ".join(temps[i:i + 12]) + ";")
        if preds:
            lines.append(".reg .pred " + ", ".join(preds) + ";")

        def o(x):
            if isinstance(x, int):
                return str(x)
            return operand.get(x, x)

        for op, dst, srcs in self.ops:
            if op == "label":
                lines.append("%s:" % dst)
            elif op == "bra_if_not":
                lines.append("@!%s bra %s;" % (dst, srcs[0]))
            elif op == "setp.lt.u32":
                lines.append("setp.lt.u32 %s, %s, %s;" % (dst, o(srcs[0]), o(srcs[1])))
            elif op.startswith("shf.l"):
                lines.append("shf.l.clamp.b32 %s, %s, %s, %s;" % (o(dst), o(srcs[0]), o(srcs[1]), o(srcs[2])))
            elif op.startswith("and"):
                lines.append("and.b32 %s, %s, %s;" % (o(dst), o(srcs[0]), o(srcs[1])))
            else:
                lines.append("%s %s, %s;" % (op, o(dst), ", ".join(o(x) for x in srcs)))
        lines.append("}")
        return lines


def chain_row(pr, arr, defined, ai, terms, first_free):
    """Accumulate products ai*bj at consecutive register pairs of `arr`.
    terms: list of (lo_index, bj_name) with lo_index increasing by 2. defined: set of indices already holding data."""
    first = True
    last_hi_defined = False
    for lo, bj in terms:
        hi = lo + 1
        lo_def, hi_def = lo in defined, hi in defined
        opl = ("mad.lo.cc.u32" if first else "madc.lo.cc.u32")
        pr.emit(opl, arr % lo, ai, bj, (arr % lo) if lo_def else 0)
        pr.emit("madc.hi.cc.u32", arr % hi, ai, bj, (arr % hi) if hi_def else 0)
        defined.add(lo)
        defined.add(hi)
        last_hi_defined = hi_def
        first = False
        top = hi
    # propagate the carry through every higher limb that already holds data, then into a fresh limb
    k = top + 1
    while k in defined:
        pr.emit("addc.cc.u32", arr % k, arr % k, 0)
        last_hi_defined = True
        k += 1
    if last_hi_defined and k < first_free:
        pr.emit("addc.u32", arr % k, 0, 0)
        defined.add(k)


def gen_fold_top(pr, c, top, tag):
    """c[0..7] += 38 * top (top < 2^7) with the carry ripple out of limb 0 — probability ~2^-21 — taken out of line."""
    pr.emit("mul.lo.u32", top, top, 38)
    pr.emit("add.u32", c[0], c[0], top)
    pr.emit("setp.lt.u32", "p_" + tag, c[0], top)          # wrapped  <=>  sum < addend
    pr.emit("bra_if_not", "p_" + tag, "L_" + tag)
    pr.emit("add.cc.u32", c[1], c[1], 1)
    for k in range(2, 8):
        pr.emit("addc.cc.u32", c[k], c[k], 0)
    pr.emit("addc.u32", "w_" + tag, 0, 0)
    # a second wrap leaves a value < 2^13 in c, so +38 cannot carry again
    pr.emit("mul.lo.u32", "w_" + tag, "w_" + tag, 38)
    pr.emit("add.u32", c[0], c[0], "w_" + tag)
    pr.emit("label", "L_" + tag)


def gen_reduce(pr, c, out):
    """c[0..15] (names) -> value = c mod p in [0, 2^256), left in c[0..7] (which must be the output names)."""
    assert list(c[:8]) == list(out)
    # even columns: (c0,c1) += 38*c8 ; (c2,c3) += 38*c10 ; ...
    first = True
    for j in (0, 2, 4, 6):
        pr.emit("mad.lo.cc.u32" if first else "madc.lo.cc.u32", c[j], c[8 + j], 38, c[j])
        pr.emit("madc.hi.cc.u32", c[j + 1], c[8 + j], 38, c[j + 1])
        first = False
    pr.emit("addc.u32", "t8", 0, 0)
    # odd columns: fresh products
    for j in (1, 3, 5, 7):
        pr.emit("mul.lo.u32", "q%d" % j, c[8 + j], 38)
        pr.emit("mul.hi.u32", "q%d" % (j + 1), c[8 + j], 38)
    pr.emit("add.cc.u32", c[1], c[1], "q1")
    for k in range(2, 8):
        pr.emit("addc.cc.u32", c[k], c[k], "q%d" % k)
    pr.emit("addc.u32", "t8", "t8", "q8")
    gen_fold_top(pr, c, "t8", "red")


def gen_reduce_split(pr, E, O, out):
    """Fold a 512-bit value held as TWO interleaved accumulator arrays — E[k] at column k (k = 0..15, even-aligned pairs)
    and O[k] at column k+1 (k = 0..14, odd-aligned pairs) — down to out[0..7] without ever re-pairing a register:
    high limbs at even columns fold (x38) into E's low pairs, high limbs at odd columns into O's low pairs, so every
    wide multiply-accumulate keeps the (even, odd) register pair it was born with (no IMAD.MOV shuffles in SASS)."""
    assert [E % k for k in range(8)] == list(out)
    h = {}
    for p in range(8, 16):
        h[p] = "h%d" % p
        op = "add.cc.u32" if p == 8 else ("addc.cc.u32" if p < 15 else "addc.u32")
        pr.emit(op, h[p], E % p, O % (p - 1))
    first = True
    for j in (0, 2, 4, 6):                                  # even columns -> E pairs (j, j+1)
        pr.emit("mad.lo.cc.u32" if first else "madc.lo.cc.u32", E % j, h[8 + j], 38, E % j)
        pr.emit("madc.hi.cc.u32", E % (j + 1), h[8 + j], 38, E % (j + 1))
        first = False
    pr.emit("addc.u32", "te", 0, 0)                          # column 8
    first = True
    for j in (1, 3, 5, 7):                                  # odd columns -> O pairs (columns j, j+1) = O[j-1], O[j]
        lo, hi = O % (j - 1), (O % j) if j < 7 else "x7"
        pr.emit("mad.lo.cc.u32" if first else "madc.lo.cc.u32", lo, h[8 + j], 38, lo)
        if j < 7:
            pr.emit("madc.hi.cc.u32", hi, h[8 + j], 38, hi)
        else:
            pr.emit("madc.hi.u32", hi, h[8 + j], 38, 0)     # column 8, fresh (O[7] was consumed by h8)
        first = False
    pr.emit("add.cc.u32", out[1], E % 1, O % 0)
    for k in range(2, 8):
        pr.emit("addc.cc.u32", out[k], E % k, O % (k - 1))
    pr.emit("addc.u32", "t8", "te", "x7")
    gen_fold_top(pr, list(out), "t8", "red")


def gen_mul():
    pr = Prog()
    a = ["a%d" % i for i in range(8)]
    b = ["b%d" % i for i in range(8)]
    class Names:                      # even accumulators 0..7 are the outputs themselves (no copy at the end)
        def __mod__(self, k):
            return ("r%d" % k) if k < 8 else ("e%d" % k)
    E, O = Names(), "o%d"      # o[k] holds column k+1
    de, do = set(), set()
    for i in range(8):
        te = [(i + j, b[j]) for j in range(8) if (i + j) % 2 == 0]
        to = [(i + j - 1, b[j]) for j in range(8) if (i + j) % 2 == 1]
        if i == 0:
            for lo, bj in te:
                pr.emit("mul.lo.u32", E % lo, a[0], bj); pr.emit("mul.hi.u32", E % (lo + 1), a[0], bj)
                de |= {lo, lo + 1}
            for lo, bj in to:
                pr.emit("mul.lo.u32", O % lo, a[0], bj); pr.emit("mul.hi.u32", O % (lo + 1), a[0], bj)
                do |= {lo, lo + 1}
            continue
        chain_row(pr, E, de, a[i], te, 16)
        chain_row(pr, O, do, a[i], to, 15)
    assert de == set(range(16)) and do == set(range(15)), (de, do)
    class ONames:
        def __mod__(self, k):
            return "o%d" % k
    gen_reduce_split(pr, E, ONames(), ["r%d" % k for k in range(8)])
    return pr


def prod4(pr, x, y, tag, out):
    """out[0..7] = x[0..3] * y[0..3] (4 x 4 limbs) through the same even/odd accumulator arrays as the 8 x 8 product (every lo/hi pair
    fuses to one IMAD.WIDE.U32[.X]); the two arrays are merged into eight plain limbs at the end."""
    class EN:
        def __mod__(self, k):
            return "%se%d" % (tag, k)
    class ON:
        def __mod__(self, k):
            return "%so%d" % (tag, k)
    E, O = EN(), ON()
    de, do = set(), set()
    for i in range(4):
        te = [(i + j, y[j]) for j in range(4) if (i + j) % 2 == 0]
        to = [(i + j - 1, y[j]) for j in range(4) if (i + j) % 2 == 1]
        if i == 0:
            for lo, bj in te:
                pr.emit("mul.lo.u32", E % lo, x[0], bj); pr.emit("mul.hi.u32", E % (lo + 1), x[0], bj)
                de |= {lo, lo + 1}
            for lo, bj in to:
                pr.emit("mul.lo.u32", O % lo, x[0], bj); pr.emit("mul.hi.u32", O % (lo + 1), x[0], bj)
                do |= {lo, lo + 1}
            continue
        chain_row(pr, E, de, x[i], te, 8)
        chain_row(pr, O, do, x[i], to, 7)
    assert de == set(range(8)) and do == set(range(7)), (de, do)
    pr.emit("add.u32", out[0], E % 0, 0)
    pr.emit("add.cc.u32", out[1], E % 1, O % 0)
    for k in range(2, 7):
        pr.emit("addc.cc.u32", out[k], E % k, O % (k - 1))
    pr.emit("addc.u32", out[7], E % 7, O % 6)


def gen_mul_karatsuba():
    """One level of Karatsuba on 4-limb halves: 3 x 16 = 48 wide multiplies instead of 64 (+ 8 for the fold), paid for with ~80 more
    adds / subtracts on the ALU pipe — the pipe that has slack in k_verify_main (31 % busy against 83 % for the multiply pipe).
    MEASURED AND NOT KEPT (round 2): correct (simulation + GPU parity), but the mixed-addition loop grows from 1,120 to 1,562 SASS
    instructions (the three short products triple the carry materialisations: 164 IMAD.MOV + 157 SEL) and k_verify_main takes
    2.44 ms instead of 2.26 ms per 2^20.  Emitted into fe_asm.cuh only with HS_GEN_KARATSUBA=1 (fe.cuh: -DHS_FE_KARATSUBA)."""
    pr = Prog()
    a = ["a%d" % i for i in range(8)]
    b = ["b%d" % i for i in range(8)]
    sa, sb = ["sa%d" % i for i in range(4)], ["sb%d" % i for i in range(4)]
    for s_, x, c in ((sa, a, "ca"), (sb, b, "cb")):
        pr.emit("add.cc.u32", s_[0], x[0], x[4])
        for k in range(1, 4):
            pr.emit("addc.cc.u32", s_[k], x[k], x[k + 4])
        pr.emit("addc.u32", c, 0, 0)
    p0 = ["r0", "r1", "r2", "r3", "p04", "p05", "p06", "p07"]
    p2 = ["p2%d" % k for k in range(8)]
    pm = ["pm%d" % k for k in range(9)]
    prod4(pr, a[:4], b[:4], "x", p0)
    prod4(pr, a[4:], b[4:], "y", p2)
    prod4(pr, sa, sb, "z", pm[:8])
    # (sa + ca 2^128)(sb + cb 2^128) = pm + (ca sb + cb sa) 2^128 + ca cb 2^256
    pr.emit("sub.u32", "ma", 0, "ca")
    pr.emit("sub.u32", "mb", 0, "cb")
    for k in range(4):
        pr.emit("and", "ta%d" % k, sb[k], "ma")
        pr.emit("and", "tb%d" % k, sa[k], "mb")
    pr.emit("add.cc.u32", pm[4], pm[4], "ta0")
    for k in range(1, 4):
        pr.emit("addc.cc.u32", pm[4 + k], pm[4 + k], "ta%d" % k)
    pr.emit("addc.u32", pm[8], 0, 0)
    pr.emit("add.cc.u32", pm[4], pm[4], "tb0")
    for k in range(1, 4):
        pr.emit("addc.cc.u32", pm[4 + k], pm[4 + k], "tb%d" % k)
    pr.emit("addc.u32", pm[8], pm[8], 0)
    pr.emit("and", "cab", "ca", "cb")
    pr.emit("add.u32", pm[8], pm[8], "cab")
    # middle term = that - p0 - p2 (non-negative, < 2^258)
    for sub in (p0, p2):
        pr.emit("sub.cc.u32", pm[0], pm[0], sub[0])
        for k in range(1, 8):
            pr.emit("subc.cc.u32", pm[k], pm[k], sub[k])
        pr.emit("subc.u32", pm[8], pm[8], 0)
    # c[0..15] = p0 + middle 2^128 + p2 2^256
    c = ["r%d" % k for k in range(8)] + ["c%d" % k for k in range(8, 16)]
    pr.emit("add.cc.u32", c[4], p0[4], pm[0])
    for k in range(1, 4):
        pr.emit("addc.cc.u32", c[4 + k], p0[4 + k], pm[k])
    for k in range(4):
        pr.emit("addc.cc.u32", c[8 + k], p2[k], pm[4 + k])
    pr.emit("addc.cc.u32", c[12], p2[4], pm[8])
    pr.emit("addc.cc.u32", c[13], p2[5], 0)
    pr.emit("addc.cc.u32", c[14], p2[6], 0)
    pr.emit("addc.u32", c[15], p2[7], 0)
    gen_reduce(pr, c, c[:8])
    return pr


def gen_sqr(split=True):
    pr = Prog()
    a = ["a%d" % i for i in range(8)]
    E, O = "e%d", "o%d"
    de, do = set(), set()
    for i in range(7):
        te = [(i + j, a[j]) for j in range(i + 1, 8) if (i + j) % 2 == 0]
        to = [(i + j - 1, a[j]) for j in range(i + 1, 8) if (i + j) % 2 == 1]
        for arr, dset, terms, lim in ((E, de, te, 16), (O, do, to, 15)):
            if not terms:
                continue
            if terms[0][0] not in dset and all(x not in dset for t in terms for x in (t[0], t[0] + 1)):
                for lo, bj in terms:
                    pr.emit("mul.lo.u32", arr % lo, a[i], bj); pr.emit("mul.hi.u32", arr % (lo + 1), a[i], bj)
                    dset |= {lo, lo + 1}
            else:
                chain_row(pr, arr, dset, a[i], terms, lim)
    if not split:
        # off-diagonal sum S occupies columns 1..14 (< 2^511); e covers even-aligned pairs, o odd-aligned
        # c[k] = e[k] + o[k-1] for k in 0..15 (missing -> 0)
        c = []
        first = True
        for k in range(16):
            ek = (E % k) if k in de else None
            ok = (O % (k - 1)) if (k - 1) in do else None
            name = ("r%d" % k) if k < 8 else ("c%d" % k)
            if ek is None and ok is None:
                pr.emit("add.u32", name, 0, 0) if first else pr.emit("addc.cc.u32", name, 0, 0)
            elif first:
                if ek is not None and ok is not None:
                    pr.emit("add.cc.u32", name, ek, ok); first = False
                else:
                    pr.emit("add.u32", name, ek if ek is not None else ok, 0)
            else:
                pr.emit("addc.cc.u32", name, ek if ek is not None else 0, ok if ok is not None else 0)
            c.append(name)
        for k in range(15, 0, -1):
            pr.emit("shf.l", c[k], c[k - 1], c[k], 1)
        pr.emit("shf.l", c[0], 0, c[0], 1)
        for i in range(8):
            pr.emit("mad.lo.cc.u32" if i == 0 else "madc.lo.cc.u32", c[2 * i], a[i], a[i], c[2 * i])
            pr.emit("madc.hi.cc.u32", c[2 * i + 1], a[i], a[i], c[2 * i + 1])
        gen_reduce(pr, c, ["r%d" % k for k in range(8)])
        return pr
    # off-diagonal sum S = E + (O << 32) occupies columns 1..14 (< 2^511).  2S = 2E + (2O << 32): double each array on its
    # own (the arrays never merge, so no register changes its pair), then add the diagonal a_i^2 at column 2i into E's pairs.
    class EN:
        def __mod__(self, k):
            return ("r%d" % k) if k < 8 else ("f%d" % k)
    class ON:
        def __mod__(self, k):
            return "g%d" % k
    NE, NO = EN(), ON()
    for arr, dset, new, n in ((E, de, NE, 16), (O, do, NO, 15)):
        for k in range(n - 1, -1, -1):
            cur = (arr % k) if k in dset else None
            prev = (arr % (k - 1)) if (k - 1) in dset else None
            if cur is None and prev is None:
                pr.emit("add.u32", new % k, 0, 0)
            elif prev is None:
                pr.emit("add.u32", new % k, cur, cur)            # low limb of a run: plain shift left by one
            elif cur is None:
                pr.emit("shf.l", new % k, prev, 0, 1)            # only the bit shifted out of the limb below
            else:
                pr.emit("shf.l", new % k, prev, cur, 1)
    for i in range(8):
        pr.emit("mad.lo.cc.u32" if i == 0 else "madc.lo.cc.u32", NE % (2 * i), a[i], a[i], NE % (2 * i))
        pr.emit("madc.hi.cc.u32" if i < 7 else "madc.hi.u32", NE % (2 * i + 1), a[i], a[i], NE % (2 * i + 1))
    gen_reduce_split(pr, NE, NO, ["r%d" % k for k in range(8)])
    return pr


def gen_add():
    """r = a + b mod p (result in [0, 2^256)): 8-limb add, fold the carry as +38, rare second ripple out of line."""
    pr = Prog()
    pr.emit("add.cc.u32", "r0", "a0", "b0")
    for k in range(1, 8):
        pr.emit("addc.cc.u32", "r%d" % k, "a%d" % k, "b%d" % k)
    pr.emit("addc.u32", "t8", 0, 0)
    gen_fold_top(pr, ["r%d" % k for k in range(8)], "t8", "add")
    return pr


def gen_sub():
    """r = a - b mod p: 8-limb subtract, fold the borrow as -38, rare second ripple out of line."""
    pr = Prog()
    pr.emit("sub.cc.u32", "r0", "a0", "b0")
    for k in range(1, 8):
        pr.emit("subc.cc.u32", "r%d" % k, "a%d" % k, "b%d" % k)
    pr.emit("subc.u32", "t8", 0, 0)              # 0 or 0xffffffff
    pr.emit("and", "t8", "t8", 38)
    pr.emit("setp.lt.u32", "p_sub", "r0", "t8")  # the -38 borrows out of limb 0 (probability ~2^-27)
    pr.emit("sub.u32", "r0", "r0", "t8")
    pr.emit("bra_if_not", "p_sub", "L_sub")
    pr.emit("sub.cc.u32", "r1", "r1", 1)
    for k in range(2, 8):
        pr.emit("subc.cc.u32", "r%d" % k, "r%d" % k, 0)
    pr.emit("subc.u32", "w_sub", 0, 0)
    pr.emit("and", "w_sub", "w_sub", 38)
    pr.emit("sub.u32", "r0", "r0", "w_sub")      # after a second wrap the value is >= 2^256-38: no further borrow
    pr.emit("label", "L_sub")
    return pr


def check_addsub(pr, is_sub):
    rnd = random.Random(99)
    top = (1 << 256) - 1
    specials = [0, 1, 37, 38, 39, P - 1, P, P + 1, 2 * P, 2 * P + 1, top, top - 37, top - 38, (1 << 255), M32, M32 - 37, (top ^ M32), (top ^ M32) + 5,
                (1 << 32), (1 << 32) + 37, (1 << 224)]
    cases = [(x, y) for x in specials for y in specials]
    for _ in range(4000):
        x, y = rnd.getrandbits(256), rnd.getrandbits(256)
        if rnd.random() < 0.3:
            y = (top - x + rnd.randrange(-60, 60)) & top if not is_sub else (x + rnd.randrange(-60, 60)) & top
        cases.append((x, y))
    # crafted: the ripple alone (the folded low limb carries or borrows, the limbs above do not all pass it on) and the second wrap
    # (a + b within 38 of 2^257 for add; a - b within 38 of -2^256 for sub)
    for _ in range(200):
        hi = rnd.getrandbits(224) << 32
        if is_sub:
            x = rnd.randrange(37)
            cases.append((x, (x - hi - rnd.randrange(38)) % (1 << 256)))              # (x - y) mod 2^256 = hi + (< 38), hi != 0
            cases.append((x, top - rnd.randrange(37 - x)))                              # x - y + 2^256 - 38 < 0
        else:
            cases.append((hi | (M32 - rnd.randrange(38)), top - hi))                   # sum = 2^256 + (< 2^32), within 38 of 2^256 + 2^32
            x = top - rnd.randrange(19)
            cases.append((x, top - rnd.randrange(19)))                                 # sum > 2^257 - 38
    ripples = wraps = 0
    tag = "sub" if is_sub else "add"
    for x, y in cases:
        env = {"a%d" % i: v for i, v in enumerate(limbs(x))}
        env.update({"b%d" % i: v for i, v in enumerate(limbs(y))})
        trace = set()
        out = pr.run(env, trace)
        r = sum(out["r%d" % i] << (32 * i) for i in range(8))
        assert r < (1 << 256) and r % P == ((x - y) if is_sub else (x + y)) % P, (hex(x), hex(y), hex(r))
        ripples += ("L_" + tag) in trace
        wraps += out.get("w_" + tag, 0) != 0
    assert ripples >= 300 and wraps >= 150, ("%s: ripple / second wrap too rarely taken" % tag, ripples, wraps)


def check_reduce_split():
    """gen_reduce_split on arbitrary (E, O) pairs with E + (O << 32) < 2^512, including rare-ripple inputs."""
    class EN:
        def __mod__(self, k):
            return ("r%d" % k) if k < 8 else ("e%d" % k)
    class ON:
        def __mod__(self, k):
            return "o%d" % k
    pr = Prog()
    gen_reduce_split(pr, EN(), ON(), ["r%d" % k for k in range(8)])
    rnd = random.Random(11)
    trace = set()
    cases = []
    for _ in range(4000):
        v = rnd.getrandbits(512) if rnd.random() < 0.7 else (1 << 512) - 1 - rnd.getrandbits(rnd.randrange(1, 200))
        o = rnd.getrandbits(480) if rnd.random() < 0.8 else (1 << 480) - 1
        o = min(o, v >> 32)
        cases.append((v - (o << 32), o))
    for _ in range(3000):   # engineered: result just below 2^256 before the last fold
        hi = rnd.getrandbits(256)
        lo = (((1 << 256) - rnd.randrange(1, 3000)) - 38 * hi) % (1 << 256)
        v = (hi << 256) | lo
        o = rnd.getrandbits(480)
        o = min(o, v >> 32)
        cases.append((v - (o << 32), o))
    for e, o in cases:
        env = {EN() % k: (e >> (32 * k)) & M32 for k in range(16)}
        env.update({"o%d" % k: (o >> (32 * k)) & M32 for k in range(15)})
        out = pr.run(env, trace)
        r = sum(out["r%d" % i] << (32 * i) for i in range(8))
        assert r < (1 << 256) and r % P == (e + (o << 32)) % P, (hex(e), hex(o))
    assert "L_red" in trace, "split-reduce ripple never exercised"


def check_reduce():
    """gen_reduce on arbitrary 512-bit inputs, including ones built to hit the out-of-line ripple."""
    pr = Prog()
    c = ["r%d" % k for k in range(8)] + ["e%d" % k for k in range(8, 16)]
    gen_reduce(pr, c, c[:8])
    check_reduce_split()
    rnd = random.Random(7)
    trace = set()
    cases = [rnd.getrandbits(512) for _ in range(3000)] + [(1 << 512) - 1, 0, (1 << 256) - 1, ((1 << 256) - 1) << 256]
    for _ in range(3000):   # low limb close to wrapping after the fold, upper limbs all ones -> long ripple
        hi = rnd.getrandbits(256)
        lo_target = ((1 << 256) - rnd.randrange(1, 3000)) & ((1 << 256) - 1)
        lo = (lo_target - 38 * hi) % (1 << 256)
        cases.append((hi << 256) | lo)
    for v in cases:
        env = {name: (v >> (32 * k)) & M32 for k, name in enumerate(c)}
        out = pr.run(env, trace)
        r = sum(out["r%d" % i] << (32 * i) for i in range(8))
        assert r < (1 << 256) and r % P == v % P, hex(v)
    assert "L_red" in trace, "reduce ripple never exercised"


def limbs(v, n=8):
    return [(v >> (32 * i)) & M32 for i in range(n)]


def crafted_products(rnd, n):
    """Products that take the out-of-line ripple of the final fold and, mostly, its second wrap: with M = 2p = 2^256 - 38, a odd and
    b = s a^-1 mod M for a small s in [39, 75], a * b = s + j M.  The first fold leaves s + q M for a small q, and when q >= 2 that is
    (q - 1) 2^256 + (2^256 + s - 38 q): limbs 1..7 all ones, so the final +38 (q - 1) carries out of every limb and wraps to s."""
    out = []
    while len(out) < n:
        a = rnd.getrandbits(256) | 1
        if a % P:
            out.append((a, rnd.randrange(39, 76) * pow(a, -1, 2 * P) % (2 * P)))
    return out


def crafted_squares():
    """The same for squares: a = sqrt(s) mod p for the squares s in [39, 200), its parity chosen so that a^2 = s mod 2p."""
    out = []
    for s in range(39, 200):
        if pow(s, (P - 1) // 2, P) != 1:
            continue
        x = pow(s, (P + 3) // 8, P)
        if x * x % P != s:
            x = x * pow(2, (P - 1) // 4, P) % P
        for a in (x, P - x):
            out.append(a + P if a % 2 == 0 else a)
    return out


def check(pr, is_sqr):
    """pr against Python integers on specials, random and crafted inputs; the crafted ones must take the fold's ripple and second
    wrap often enough that both out-of-line paths are proven, not just present."""
    rnd = random.Random(1234)
    specials = [0, 1, 2, P - 1, P, P + 1, 2 * P, 2 * P + 1, (1 << 256) - 1, (1 << 256) - 38, (1 << 256) - 39,
                (1 << 255), (1 << 255) - 1, M32, M32 << 224, int("f" * 8 + "0" * 8, 16) * ((1 << 256) // ((1 << 64) - 1))]
    cases = [(x, y) for x in specials for y in specials]
    for _ in range(3000):
        x = rnd.getrandbits(256); y = rnd.getrandbits(256)
        if rnd.random() < 0.3:
            x |= ((1 << 256) - 1) ^ ((1 << rnd.randrange(256)) - 1)
        if rnd.random() < 0.3:
            y = ((1 << 256) - 1) >> rnd.randrange(64)
        cases.append((x, y))
    cases += [(a, a) for a in crafted_squares()] if is_sqr else crafted_products(rnd, 200)
    ripples = wraps = 0
    for x, y in cases:
        if is_sqr:
            y = x
        env = {"a%d" % i: v for i, v in enumerate(limbs(x))}
        env.update({"b%d" % i: v for i, v in enumerate(limbs(y))})
        trace = set()
        out = pr.run(env, trace)
        r = sum(out["r%d" % i] << (32 * i) for i in range(8))
        assert r < (1 << 256)
        assert r % P == (x * y) % P, (hex(x), hex(y), hex(r))
        ripples += "L_red" in trace
        wraps += out.get("w_red", 0) != 0
    assert ripples >= (40 if is_sqr else 150) and wraps >= (40 if is_sqr else 150), ("fold ripple / second wrap too rarely taken", ripples, wraps)


def emit_function(name, pr, nin):
    # asm volatile is not needed: the block has no side effects beyond its outputs
    operand = {}
    idx = 0
    for k in range(8):
        operand["r%d" % k] = "%%%d" % idx; idx += 1
    for k in range(8):
        operand["a%d" % k] = "%%%d" % idx; idx += 1
    if nin == 2:
        for k in range(8):
            operand["b%d" % k] = "%%%d" % idx; idx += 1
    lines = pr.ptx(operand)
    body = "\n".join('      "%s\\n\\t"' % ln for ln in lines)
    outs = ", ".join('"=&r"(r[%d])' % k for k in range(8))
    ins = ", ".join('"r"(a[%d])' % k for k in range(8))
    if nin == 2:
        ins += ", " + ", ".join('"r"(b[%d])' % k for k in range(8))
        sig = "uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]"
    else:
        sig = "uint32_t (&r)[8], const uint32_t (&a)[8]"
    return ("__device__ __forceinline__ void %s(%s) {\n  asm(\n%s\n      : %s\n      : %s);\n}\n" % (name, sig, body, outs, ins))


def count(pr):
    w = sum(1 for op, _, _ in pr.ops if ".hi" in op)          # each lo/hi pair fuses into one IMAD.WIDE
    other = sum(1 for op, _, _ in pr.ops if not op.startswith(("mul", "mad")))
    return w, other


def render(sqr_split=True, karatsuba=False):
    """Generate every sequence, run every check above on it, and return the text of fe_asm.cuh (the committed file is this text:
    tests/test_device_arith_edges.py compares them byte for byte).  karatsuba: also emit fe_mul_karatsuba_asm."""
    m, s = gen_mul(), gen_sqr(split=sqr_split)
    mk = gen_mul_karatsuba()   # experiment (the three short products triple the carry materialisations); emitted only on request
    check(mk, False)
    check(m, False)
    check(s, True)
    check_reduce()
    ad, sb = gen_add(), gen_sub()
    check_addsub(ad, False)
    check_addsub(sb, True)
    hdr = ("// GENERATED by tools/gen_fe_asm.py — do not edit.\n"
           "// GF(2^255-19) multiply / square on 8 saturated 32-bit limbs; mad.lo.cc/madc.hi.cc pairs fuse to IMAD.WIDE.U32.X.\n"
           "// Every sequence below was simulated against Python big integers by the generator before being emitted.\n"
           "#pragma once\n#include <cstdint>\n\n")
    return (hdr + emit_function("fe_mul_asm", m, 2) + "\n" + (emit_function("fe_mul_karatsuba_asm", mk, 2) + "\n" if karatsuba else "") + emit_function("fe_sqr_asm", s, 1) + "\n" +
            emit_function("fe_add_asm", ad, 2) + "\n" + emit_function("fe_sub_asm", sb, 2))


if __name__ == "__main__":
    txt = render(sqr_split=os.environ.get('HS_SQR_SPLIT', '1') == '1', karatsuba=os.environ.get("HS_GEN_KARATSUBA") == "1")
    path = os.path.join(ROOT, "hotstuff_b200", "csrc", "fe_asm.cuh")
    open(path, "w").write(txt)
    m, mk, s = gen_mul(), gen_mul_karatsuba(), gen_sqr(split=os.environ.get('HS_SQR_SPLIT', '1') == '1')
    print("mul: %d wide-mads + %d other ops; karatsuba mul: %d + %d; sqr: %d wide-mads + %d other ops -> %s" % (count(m) + count(mk) + count(s) + (path,)))
