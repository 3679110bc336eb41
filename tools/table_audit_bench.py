#!/usr/bin/env python3
"""Cost of hs_table_audit (hotstuff_b200.Engine.table_audit), and whether an audit in flight moves a vote burst's latency.

Workloads (each a fresh context; committees of keys from seeds, registered as a node would):
  keys4096_w13   4,096 keys at 13-bit key windows (the window an 80 GB H100 picks for that committee), 24-bit base table
  keys10000_w12  10,000 keys at 12-bit key windows, 24-bit base table
  keys64         64 keys at the window registration picks (the base table dominates the work)
  base_w24       a fresh context: the 24-bit base table alone
  base_w26       a fresh context: the 26-bit base table alone
Time per call: host clock around the returning call (it ends in a stream synchronise), median of --reps after one warm-up call.
Rates are computed from shapes: every entry is read once (96 bytes) and costs about 12 field multiplications (3 for its third
coordinate, 9 for the step from the previous entry).  "bound" names the resource the measured rates point at: HBM when the bytes rate is
at least half the data-sheet 3.35 TB/s, otherwise the multiply pipe.
Burst: on the 4,096-key context, 667 single-vote requests from 16 threads through one verify queue; the p50 of their submit-to-verdict
latencies without and with audits running back to back in another thread, alternated --reps times.
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run (the SM clock
also sampled while an audit runs).

    python tools/table_audit_bench.py [--reps 5] [--out profiles/r02_table_audit.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ENTRY_BYTES = 96
MULS_PER_ENTRY = 12
HBM_BYTES_PER_S = 3.35e12  # NVIDIA data sheet, H100 SXM


def smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unavailable"


def ndigits(w):
    r = 253 % w
    return (253 + w - 1) // w + (1 if r in (0, w - 1) else 0)


def entries(w):
    return ndigits(w) * ((1 << (w - 1)) + 1)


def keys(eng, n, seed):
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    return seeds, eng.keygen_batch(seeds)


def time_audit(eng, reps):
    failed, _ = eng.table_audit()
    assert failed == 0, eng.last_error
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        failed, _ = eng.table_audit()
        ts.append(time.perf_counter() - t0)
        assert failed == 0, eng.last_error
    return statistics.median(ts), ts


def shape_line(name, eng, med, ts, card):
    wa, wb = eng.window_bits
    n = eng.key_slots
    ent = n * (entries(wa) if n else 0) + entries(wb)
    byts, muls = ent * ENTRY_BYTES, ent * MULS_PER_ENTRY
    return {"workload": name, "key_slots": n, "key_window": wa if n else 0, "base_window": wb, "entries": ent, "bytes": byts,
            "audit_ms_median": round(med * 1e3, 3), "audit_ms_all": [round(t * 1e3, 3) for t in ts],
            "entries_per_s": round(ent / med, 1), "field_muls_per_s": round(muls / med, 1), "bytes_per_s": round(byts / med, 1),
            "hbm_share_of_datasheet": round(byts / med / HBM_BYTES_PER_S, 4),
            "bound": "HBM" if byts / med >= 0.5 * HBM_BYTES_PER_S else "multiply pipe", "card": card}


def burst(q, recs, threads=16):
    lat = [0.0] * len(recs)
    out = [None] * len(recs)

    def worker(t):
        for i in range(t, len(recs), threads):
            t0 = time.perf_counter()
            out[i] = q.wait(q.submit(recs[i:i + 1]))[0]
            lat[i] = time.perf_counter() - t0

    th = [threading.Thread(target=worker, args=(t,)) for t in range(threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return statistics.median(lat), np.array(out, bool)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_table_audit.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("table_audit_bench: no GPU")
    from hotstuff_b200 import Engine
    card = smi()
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    for name, n, kw, bw in (("keys4096_w13", 4096, 13, 0), ("keys10000_w12", 10000, 12, 0), ("keys64", 64, 0, 0), ("base_w24", 0, 0, 24),
                            ("base_w26", 0, 0, 26)):
        eng = Engine(0, base_window=bw, key_window=kw)
        try:
            if n:
                seeds, pks = keys(eng, n, n)
                eng.committee_register(pks)
                failed, _ = eng.table_audit(pks)
                assert failed == 0, eng.last_error
            med, ts = time_audit(eng, args.reps)
            sample = {}
            th = threading.Thread(target=lambda: sample.setdefault("smi", [smi() for _ in range(3)]))
            done = threading.Event()

            def loop():
                while not done.is_set():
                    eng.table_audit()

            a = threading.Thread(target=loop)
            a.start()
            th.start()
            th.join()
            done.set()
            a.join()
            d = shape_line(name, eng, med, ts, card)
            d["smi_during_audit"] = sample["smi"]
            emit(d)
            if name == "keys4096_w13":
                emit(vote_burst(eng, seeds, pks, args.reps, card))
        finally:
            eng.close()
    if args.out:
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


def vote_burst(eng, seeds, pks, reps, card):
    """Votes signed by committee members: every record takes the queue's committee path."""
    rng = np.random.default_rng(7)
    n = 667
    ki = rng.integers(0, len(pks), n).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64] = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    recs[:, 64:96] = pks[ki]
    recs[:, 96:] = dig
    want = eng.verify_rec128(recs)
    q = eng.queue()
    try:
        burst(q, recs)  # warm-up
        quiet, busy, audits = [], [], []
        for _ in range(reps):
            p50, got = burst(q, recs)
            assert np.array_equal(got, want)
            quiet.append(p50)
            done = threading.Event()
            count = [0]

            def loop():
                while not done.is_set():
                    eng.table_audit()
                    count[0] += 1

            a = threading.Thread(target=loop)
            a.start()
            time.sleep(0.005)
            p50, got = burst(q, recs)
            done.set()
            a.join()
            assert np.array_equal(got, want)
            busy.append(p50)
            audits.append(count[0])
    finally:
        q.close()
    return {"workload": "vote_burst_667x16", "committee_keys": len(pks), "requests": n, "threads": 16,
            "p50_ms_without_audit": round(statistics.median(quiet) * 1e3, 4), "p50_ms_with_audit": round(statistics.median(busy) * 1e3, 4),
            "p50_ms_without_all": [round(x * 1e3, 4) for x in quiet], "p50_ms_with_all": [round(x * 1e3, 4) for x in busy],
            "audits_completed_per_burst": audits, "card": card}


if __name__ == "__main__":
    main()
