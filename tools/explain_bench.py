#!/usr/bin/env python3
"""Cost of hs_explain_rec128 (hotstuff_b200.Engine.explain), the table-free re-check of rejected records.

Records: seeded valid signatures over 64 keys with one bit flipped in every record, so every record is a rejected one (the records the
call exists for).  The re-check's work does not depend on the verdict: every record that parses costs two 256-bit scalar
multiplications by a radix-16 window, three doublings each for A and R, and a SHA-512 block.
Sizes: n = 1, 64, 4,096 and 65,536 records per call, on one context with the default geometry, no committee and no key cache (the
call reads no table anyway).
Time per call: host clock around the returning call (it ends in a stream synchronise, so the staging copy, the kernel and the readback
are all inside), median of --reps calls after --warmup calls of the same size.
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/explain_bench.py [--reps 30] [--warmup 5] [--out profiles/r02_explain.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIZES = (1, 64, 4096, 65536)


def smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unavailable"


def rejected_records(eng, n, seed=7):
    """n records signed on the GPU, each with one seeded bit flipped anywhere in sig | pk | msg."""
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * 64), np.uint8).reshape(64, 32).copy()
    pks = eng.keygen_batch(seeds)
    ki = (np.arange(n) % 64).astype(np.uint32)
    digests = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    recs = np.concatenate([eng.sign_digests(seeds, pks, digests, ki), pks[ki], digests], axis=1)
    bits = rng.integers(0, 128 * 8, n)
    recs[np.arange(n), bits >> 3] ^= (1 << (bits & 7)).astype(np.uint8)
    return np.ascontiguousarray(recs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_explain.jsonl"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("explain_bench: no CUDA device (a time measured without the GPU means nothing)")
    from hotstuff_b200 import Engine
    card = smi()
    eng = Engine(0, key_cache=False)
    recs = rejected_records(eng, max(SIZES))
    assert not eng.verify_rec128(recs, 1).any(), "a flipped bit left a record valid"
    lines = []
    for n in SIZES:
        r = np.ascontiguousarray(recs[:n])
        for _ in range(a.warmup):
            why = eng.explain(r)
        assert (why != 0).all()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            eng.explain(r)
            ts.append(time.perf_counter() - t0)
        med = statistics.median(ts)
        lines.append({"bench": "hs_explain_rec128", "n": n, "median_ms": round(med * 1e3, 4), "min_ms": round(min(ts) * 1e3, 4),
                      "max_ms": round(max(ts) * 1e3, 4), "us_per_record": round(med * 1e6 / n, 3), "reps": a.reps, "warmup": a.warmup,
                      "timing": "host clock around the returning call", "gpu": card})
        print(json.dumps(lines[-1]), flush=True)
    eng.close()
    lines.append({"bench": "card_after", "gpu": smi()})
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
