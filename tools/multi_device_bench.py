#!/usr/bin/env python3
"""Host-pointer verify calls through one context against a multi-device context (hs_multi_*, hotstuff_b200.MultiEngine).

Arms, alternated inside every repetition so that drift on a shared host hits all of them:
  single  Engine(0)
  all     MultiEngine over every visible GPU (one member on a one-GPU machine: the routing layer alone)
  00      MultiEngine([0, 0]): two members on GPU 0 (on one GPU this shows the orchestration overhead, not scaling)
Every arm has the default 24-bit base window, 12-bit key windows and the same registered 1,024-key committee; every output of every arm
is checked against the single context's before anything is timed.  Workloads:
  msgs     2^20 records of 512-byte messages through verify_msgs, key bytes, from hs_host_alloc (pinned) memory, 1 % corrupted
  groups   a 10^6-vote certificate burst through verify_groups: 1,000 Blocks, each an author signature (strict, 200-byte preimage) and a
           1,000-vote QC (batch-eq, 40-byte preimage)
  fanout   verify_rec128 at 4,096 .. 32,768 records: the cost of splitting a call.  [0, 0] shards from 2 x HS_MULTI_MIN_SHARD = 8,192
           records on; below that it runs whole on one member.
Prints one JSON line per workload and size with the card's name and power limit read in the same run (median, min, max over the
repetitions, host clock around calls that return after their results are on the host).

    python tools/multi_device_bench.py [--reps 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
COMMITTEE = 1024
KEY_WINDOW = 12


def card():
    import torch
    q = []
    for d in range(torch.cuda.device_count()):
        try:
            q.append(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(d)],
                                    capture_output=True, text=True, timeout=30).stdout.strip() or "unavailable")
        except (OSError, subprocess.SubprocessError):
            q.append("unavailable")
    return {"gpu": torch.cuda.get_device_name(0), "gpus": torch.cuda.device_count(), "nvidia_smi": q}


def pinned(lib, shape, dtype, keep):
    """A numpy array over hs_host_alloc memory (freed at exit through `keep`)."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = lib.hs_host_alloc(n)
    assert p, "hs_host_alloc(%d) failed" % n
    keep.append(p)
    return np.frombuffer((ctypes.c_uint8 * n).from_address(p), dtype=dtype).reshape(shape)


def stat(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4), "max": round(float(np.max(v)), 4)}


def timed(arms, reps, call, inner=1):
    """call(arm) per arm, alternating, reps times; ms per call."""
    out = {name: [] for name in arms}
    for _ in range(reps):
        for name, a in arms.items():
            t0 = time.perf_counter()
            for _ in range(inner):
                call(a)
            out[name].append((time.perf_counter() - t0) * 1e3 / inner)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("multi_device_bench: needs a CUDA device")
    from hotstuff_b200 import Engine, MultiEngine
    info = card()
    sink = open(args.out, "a") if args.out else None

    def emit(d):
        line = json.dumps(dict(info, **d))
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")
            sink.flush()

    rng = np.random.default_rng(2026)
    single = Engine(0, key_window=KEY_WINDOW)
    lib = single.lib
    arms = {"single": single, "all": MultiEngine(list(range(torch.cuda.device_count())), key_window=KEY_WINDOW),
            "00": MultiEngine([0, 0], key_window=KEY_WINDOW)}
    seeds = rng.integers(0, 256, (COMMITTEE, 32), dtype=np.uint8)
    pks = single.keygen_batch(seeds)
    assert single.committee_register(pks).all()
    for name in ("all", "00"):
        assert arms[name].register_committee(pks).all()
    keep = []
    try:
        # ---- msgs: 2^20 x 512 B from pinned memory
        n, L = 1 << 20, 512
        msgs = pinned(lib, (n, L), np.uint8, keep)
        msgs[:] = rng.integers(0, 256, (n, L), dtype=np.uint8)
        kidx = rng.integers(0, COMMITTEE, n).astype(np.uint32)
        dg = single.digest32_batch(msgs.reshape(-1), np.arange(n + 1, dtype=np.uint64) * L)
        sig = pinned(lib, (n, 64), np.uint8, keep)
        sig[:] = single.sign_digests(seeds, pks, dg, key_idx=kidx)
        bad = rng.choice(n, n // 100, replace=False)
        sig[bad, 7] ^= 1
        pk = pinned(lib, (n, 32), np.uint8, keep)
        pk[:] = pks[kidx]
        call = lambda a: a.verify_msgs(sig, msgs.reshape(-1), L, pk=pk)
        want = call(single)
        assert (~want).sum() == bad.size
        for a in arms.values():
            assert (call(a) == want).all(), "verify_msgs verdicts differ between arms"
        t = timed(arms, args.reps, call)
        emit(dict(workload="msgs", records=n, msg_len=L, pinned=True, ms=({k: stat(v) for k, v in t.items()}),
                  verifies_per_s={k: round(n / (np.median(v) / 1e3)) for k, v in t.items()}))

        # ---- groups: 10^6 votes
        B, V = 1000, 1000
        pre = bytearray()
        for b in range(B):
            pre += rng.bytes(200) + rng.bytes(32) + (b + 7).to_bytes(8, "little")  # Block preimage, then its QC's hash || round
        pre = np.frombuffer(bytes(pre), np.uint8).copy()
        off = np.zeros(2 * B + 1, np.uint64)
        off[1::2] = np.arange(B, dtype=np.uint64) * 240 + 200
        off[2::2] = np.arange(1, B + 1, dtype=np.uint64) * 240
        mi = np.concatenate([[2 * b] + [2 * b + 1] * V for b in range(B)]).astype(np.uint32)
        gi = np.repeat(np.arange(B, dtype=np.uint32), V + 1)
        modes = np.tile(np.concatenate([[0], np.ones(V)]), B).astype(np.uint8)
        gk = np.concatenate([[b % COMMITTEE] + [j % COMMITTEE for j in range(V)] for b in range(B)]).astype(np.uint32)
        gdg = single.digest32_batch(pre, off)
        gsig = single.sign_digests(seeds, pks, gdg[mi], key_idx=gk)
        gbad = rng.choice(mi.size, 300, replace=False)
        gsig[gbad, 9] ^= 2
        gpk = pks[gk]
        gcall = lambda a: a.verify_groups(pre, off, gsig, mi, gi, B, mode=modes, pk=gpk, want_items=True)
        wg, wi = gcall(single)
        assert (~wi).sum() == gbad.size
        for a in arms.values():
            g, i = gcall(a)
            assert (g == wg).all() and (i == wi).all(), "verify_groups verdicts differ between arms"
        t = timed(arms, args.reps, gcall)
        emit(dict(workload="groups", items=int(mi.size), groups=B, ms={k: stat(v) for k, v in t.items()},
                  items_per_s={k: round(mi.size / (np.median(v) / 1e3)) for k, v in t.items()}))

        # ---- fan-out cost: verify_rec128 with registered keys
        recs = np.concatenate([sig[:32768], pk[:32768], dg[:32768]], axis=1)
        for m in (4096, 8192, 16384, 32768):
            r = np.ascontiguousarray(recs[:m])
            want = single.verify_rec128(r)
            for a in arms.values():
                assert (a.verify_rec128(r) == want).all(), "verify_rec128 verdicts differ between arms"
            t = timed(arms, args.reps, lambda a: a.verify_rec128(r), inner=20)
            med = {k: float(np.median(v)) for k, v in t.items()}
            emit(dict(workload="fanout", records=m, sharded_00=m // 2 >= 4096, ms={k: stat(v) for k, v in t.items()},
                      extra_ms_00_vs_single=round(med["00"] - med["single"], 4), extra_ms_all_vs_single=round(med["all"] - med["single"], 4)))
        if torch.cuda.device_count() < 2:
            emit(dict(note="one GPU visible: scaling across GPUs not measured; the 'all' arm is a one-member multi-context"))
    finally:
        for a in arms.values():
            a.close()
        for p in keep:
            lib.hs_host_free(p)
        if sink:
            sink.close()


if __name__ == "__main__":
    main()
