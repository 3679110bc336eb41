#!/usr/bin/env python3
"""Generate tests/golden/edge_digits.json — valid signatures whose comb digits reach the extreme entries of a window.

A comb window of width W holds 2^(W-1) + 1 entries: entry 0 is the identity and entry m is m * 2^(W i) * P.  The signed digit
-2^(W-1) is the only digit that gathers the last entry, and digit 0 the only one that gathers the identity; k's window-0 digit of 0
also makes the identity the first accumulator of the committee comb.  A non-top digit takes either value with probability 2^-W, so
random records almost never reach them at the widths the engine uses.  This script grinds messages until it holds, for every claim
below, one valid signature that makes it:
  k{W}:min   k = SHA-512(R || A || M) mod l has a non-top digit -2^(W-1) at key width W     (W = 8 .. 17)
  k{W}:zero  k's window-0 digit is 0 at key width W                                           (W = 8 .. 17)
  S{W}:min   S has a non-top digit -2^(W-1) at base width W                                   (W = 16, 20, 24)
  S{W}:zero  S has a non-top digit 0 at base width W                                          (W = 16, 20, 24)
Each record lists the claims it makes as "<scalar><W>:<min|zero>@<digit index>"; tests/test_device_arith_edges.py recomputes them
from the record's bytes.  Signing is the CPU oracle's (RFC 8032, deterministic), over 32-byte messages, with four keys so that the
per-key tables built for them stay small.  Only messages are ground: message j of chunk c is (c * CHUNK + j) as 32 little-endian bytes,
signed by key j % 4, and for each claim the first record in that order is kept, so the output does not depend on the process count.
Base width 24 needs about 1.7 M signatures per claim: a few minutes on 8 processes.

Run from the repo root:  python tests/golden/gen_edge_digits.py [processes]
"""
import hashlib
import json
import multiprocessing
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle_api import Oracle, L_ORDER  # noqa: E402

KEY_WIDTHS = tuple(range(8, 18))
BASE_WIDTHS = (16, 20, 24)
CHUNK = 1 << 15
N_KEYS = 4
SEEDS = [hashlib.sha256(b"hotstuff edge-digit key %d" % i).digest() for i in range(N_KEYS)]


def ndigits(w):
    """sc_ndigits_rt: the number of signed radix-2^w digits of a scalar below 2^253."""
    r = 253 % w
    return (253 + w - 1) // w + (1 if r in (0, w - 1) else 0)


def digits(s, w):
    """sc_digits_rt: digit i = bits [w i, w i + w) of s + sum_i 2^(w - 1 + w i), minus 2^(w - 1); their radix-2^w sum is s."""
    n = ndigits(w)
    u = s + sum(1 << (w - 1 + w * i) for i in range(n))
    half, mask = 1 << (w - 1), (1 << w) - 1
    return [((u >> (w * i)) & mask) - half for i in range(n)]


def k_of(sig, pk, msg):
    return int.from_bytes(hashlib.sha512(bytes(sig[:32]) + bytes(pk) + bytes(msg)).digest(), "little") % L_ORDER


def claims(sig, pk, msg):
    """Every claim the record (sig, pk, msg) makes, each with the first digit index that makes it."""
    out = []
    k, s = k_of(sig, pk, msg), int.from_bytes(bytes(sig[32:]), "little")
    for name, scalar, widths in (("k", k, KEY_WIDTHS), ("S", s, BASE_WIDTHS)):
        for w in widths:
            d = digits(scalar, w)
            half = 1 << (w - 1)
            mins = [i for i in range(len(d) - 1) if d[i] == -half]
            if mins:
                out.append("%s%d:min@%d" % (name, w, mins[0]))
            if name == "k" and d[0] == 0:
                out.append("k%d:zero@0" % w)
            if name == "S":
                zeros = [i for i in range(len(d) - 1) if d[i] == 0]
                if zeros:
                    out.append("S%d:zero@%d" % (w, zeros[0]))
    return out


def wanted():
    return ["k%d:%s" % (w, c) for w in KEY_WIDTHS for c in ("min", "zero")] + ["S%d:%s" % (w, c) for w in BASE_WIDTHS for c in ("min", "zero")]


_oracle = None
_pks = None


def _grind(chunk):
    """(chunk, [(j, sig, claims)]) for the records of one chunk that make a claim."""
    global _oracle, _pks
    if _oracle is None:
        _oracle = Oracle()
        _pks = _oracle.keygen_batch(np.frombuffer(b"".join(SEEDS), np.uint8).reshape(N_KEYS, 32))
    base = chunk * CHUNK
    msgs = np.zeros((CHUNK, 32), np.uint8)
    for b in range(8):
        msgs[:, b] = ((np.arange(base, base + CHUNK, dtype=np.uint64) >> np.uint64(8 * b)) & np.uint64(0xff)).astype(np.uint8)
    ki = np.arange(CHUNK, dtype=np.uint32) % N_KEYS
    off = np.arange(CHUNK + 1, dtype=np.uint64) * 32
    seeds = np.frombuffer(b"".join(SEEDS), np.uint8).reshape(N_KEYS, 32)
    sigs = _oracle.sign_batch(seeds, _pks, ki, msgs.reshape(-1), off, nthreads=1)
    found = []
    for j in range(CHUNK):
        c = claims(sigs[j], _pks[ki[j]], msgs[j])
        if c:
            found.append((j, sigs[j].tobytes(), c))
    return chunk, found


def main():
    procs = int(sys.argv[1]) if len(sys.argv) > 1 else (os.cpu_count() or 1)
    todo = set(wanted())
    kept = {}  # (chunk, j) -> record
    pks = Oracle().keygen_batch(np.frombuffer(b"".join(SEEDS), np.uint8).reshape(N_KEYS, 32))
    with multiprocessing.Pool(procs) as pool:
        for chunk, found in pool.imap(_grind, range(1 << 20)):   # in chunk order: the first record per claim does not depend on timing
            for j, sig, cl in found:
                new = [c for c in cl if c.split("@")[0] in todo]
                if not new:
                    continue
                todo -= {c.split("@")[0] for c in new}
                n = chunk * CHUNK + j
                kept[(chunk, j)] = {"seed": SEEDS[j % N_KEYS].hex(), "msg": n.to_bytes(32, "little").hex(), "sig": sig.hex(),
                                    "pk": pks[j % N_KEYS].tobytes().hex(), "covers": cl}
            print("chunk %d: %d claims left" % (chunk, len(todo)), flush=True)
            if not todo:
                pool.terminate()
                break
    recs = [kept[k] for k in sorted(kept)]
    doc = {"description": "Valid Ed25519 signatures over 32-byte messages whose k or S digits reach a comb window's last entry (digit "
                          "-2^(W-1)) or its identity entry (digit 0); generated by tests/golden/gen_edge_digits.py",
           "key_widths": list(KEY_WIDTHS), "base_widths": list(BASE_WIDTHS), "records": recs}
    with open(os.path.join(HERE, "edge_digits.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("%d records" % len(recs))


if __name__ == "__main__":
    main()
