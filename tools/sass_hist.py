#!/usr/bin/env python3
"""SASS opcode histogram per kernel and per loop body (backward-branch regions) of a cubin / .so.

    python tools/sass_hist.py hotstuff_b200/libhs_crypto.so k_verify_main      # kernels whose name contains the pattern
    python tools/sass_hist.py lib.so k_digest32 --loops                        # also every loop body, innermost first

Pipes (B300_MICROARCH.md "Pipe rates"): IMAD* / FFMA on the fma pipe, IADD3 / LOP3 / SHF / PRMT / ISETP / SEL on the alu pipe.
Used for before/after comparisons of the hot loop.
"""
import collections
import re
import subprocess
import sys

FMA = ("IMAD", "FFMA", "FMUL", "FADD", "HFMA2")
ALU = ("IADD3", "LOP3", "SHF", "PRMT", "ISETP", "SEL", "IABS", "LEA", "FLO", "POPC", "VOTE", "MOV", "ICMP", "BMSK", "SGXT", "IMNMX", "VIMNMX", "PLOP3", "FSEL", "IADD")


def pipe_of(op):
    base = op.split(".")[0]
    if base in FMA:
        return "fma"
    if base in ALU or base.startswith("UI") or base.startswith("UL") or base.startswith("US") or base == "UMOV":
        return "alu" if not base.startswith("U") else "uniform"
    if base in ("LDG", "STG", "LDS", "STS", "LD", "ST", "LDL", "STL", "LDC", "LDCU", "ATOMG", "RED", "LDSM"):
        return "lsu"
    if base in ("BRA", "EXIT", "BSYNC", "BSSY", "RET", "CALL", "WARPSYNC", "BAR", "NOP", "BPT", "YIELD", "DEPBAR", "ERRBAR", "MEMBAR", "NANOSLEEP", "CCTL"):
        return "ctrl"
    if base in ("SHFL", "S2R", "CS2R", "S2UR", "R2UR", "MUFU", "R2P", "P2R"):
        return "other"
    return "other"


def parse(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur is not None:
            addr = int(m.group(1), 16)
            ins = m.group(2).strip()
            ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
            cur.append((addr, ins))
    return funcs


def hist(instrs):
    h = collections.Counter()
    for _, ins in instrs:
        h[ins.split()[0]] += 1
    return h


def show(title, instrs, top=40):
    h = hist(instrs)
    pipes = collections.Counter()
    for op, c in h.items():
        pipes[pipe_of(op)] += c
    total = sum(h.values())
    print("== %s: %d instructions; pipes: %s" % (title, total, ", ".join("%s %d" % kv for kv in pipes.most_common())))
    wide = sum(c for op, c in h.items() if op.startswith("IMAD.WIDE") or op.startswith("IMAD.HI"))
    imad_other = sum(c for op, c in h.items() if op.split(".")[0] == "IMAD") - wide
    print("   wide multiplies (IMAD.WIDE*/IMAD.HI*): %d; other IMAD-pipe (IMAD.MOV/IMAD/IMAD.X/IMAD.IADD/IMAD.SHL): %d" % (wide, imad_other))
    for op, c in h.most_common(top):
        print("   %6d  %s" % (c, op))


def loops(instrs):
    out = []
    index = {a: i for i, (a, _) in enumerate(instrs)}
    for i, (a, ins) in enumerate(instrs):
        if ins.startswith("BRA"):
            m = re.search(r"0x([0-9a-f]+)", ins)
            if m:
                t = int(m.group(1), 16)
                if t <= a and t in index:
                    out.append((index[t], i))
    return sorted(set(out), key=lambda r: r[1] - r[0])


def main():
    path, pat = sys.argv[1], sys.argv[2]
    want_loops = "--loops" in sys.argv
    for name, instrs in parse(path).items():
        if pat not in name:
            continue
        show(name, instrs)
        if want_loops:
            for lo, hi in loops(instrs):
                if hi - lo < 8:
                    continue
                show("  loop body [%#x .. %#x] of %s" % (instrs[lo][0], instrs[hi][0], name[:40]), instrs[lo:hi + 1], top=25)


if __name__ == "__main__":
    main()
