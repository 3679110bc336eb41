#!/usr/bin/env python3
"""What the audit of a verify queue's signature cache (hs_queue_sig_audit) costs, and what its scrub slice does to a vote burst.

One context: a 1,024-key committee at 10-bit key windows and the default base-point table, one verify queue with the node's table
(hs_queue_sig_cache of 65,536 entries: 16,384 buckets) shared with the synchronous calls and filled by one hs_verify_rec128 pass over
65,536 valid strict records, as a node's table is after a few view changes.
  - whole: hs_queue_sig_audit over the whole table, --reps times; host clock around the synchronous call, which ends in a stream
    synchronise, so it bounds the kernel's time from above.
  - slice: 512-bucket slices (the Rust shim's SIG_AUDIT_BUCKETS_PER_TICK) walked round the table, --reps times, timed the same way.
  - burst: 667 fresh single-vote requests (cache misses, as a view change's votes are) from 16 threads through the same queue, p50 /
    p99 / max of every request's submit-to-verdict latency, verdicts checked against the oracle-equivalent engine answer.  Policies,
    alternated burst by burst, --runs bursts each: none; one 512-bucket slice every 15.6 ms (the scrub's default period) from another
    thread; 512-bucket slices back to back (the worst case).
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/sig_audit_bench.py [--reps 20] [--runs 20] [--out profiles/r02_sig_audit.jsonl]
"""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from scrub_bench import stats_ms  # noqa: E402
from table_audit_bench import keys, smi  # noqa: E402

N_KEYS, KEY_WINDOW = 1024, 10
ENTRIES = 1 << 16
SLICE = 512
PERIOD_S = 0.015625
BURST = 667


def records(eng, seeds, pks, n, seed):
    rng = np.random.default_rng(seed)
    ki = rng.integers(0, len(pks), n).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64] = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    recs[:, 64:96] = pks[ki]
    recs[:, 96:] = dig
    return recs


def burst(q, recs, want, threads=16):
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
    assert np.array_equal(np.array(out, bool), want)
    return lat


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t0)
        assert r["corrected"] == 0, r
    a = np.asarray(ts) * 1e3
    return {"median_ms": round(float(np.median(a)), 4), "min_ms": round(float(a.min()), 4), "max_ms": round(float(a.max()), 4), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_sig_audit.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("sig_audit_bench: no GPU")
    from hotstuff_b200 import Engine
    card = smi()
    lines = []

    def emit(d):
        d["card"] = card
        print(json.dumps(d), flush=True)
        lines.append(d)

    eng = Engine(0, key_window=KEY_WINDOW)
    try:
        seeds, pks = keys(eng, N_KEYS, N_KEYS)
        eng.committee_register(pks)
        q = eng.queue(ring_records=4096)
        try:
            q.sig_cache(ENTRIES)
            q.sig_share(True)
            fill = records(eng, seeds, pks, ENTRIES, 1)
            assert eng.verify_rec128(fill, 0).all()
            held = q.sig_stats()["entries_held"]
            buckets = ENTRIES // 4
            q.sig_audit()  # warm-up
            whole = timed(lambda: q.sig_audit(), args.reps)
            pos = [0]

            def one_slice():
                r = q.sig_audit(pos[0], SLICE)
                pos[0] = (pos[0] + SLICE) % buckets
                return r

            sl = timed(one_slice, args.reps)
            r = q.sig_audit()
            emit({"workload": "sig_audit_cost", "entries": ENTRIES, "buckets": buckets, "held": held, "held_audited": r["held"],
                  "whole_table": whole, "slice_buckets": SLICE, "slice": sl, "sms": torch.cuda.get_device_properties(0).multi_processor_count})

            policies = ("none", "slice_every_15.6ms", "slices_back_to_back")
            q.sig_share(False)  # the answers below are computed without touching the table: the bursts' votes are misses
            votes = records(eng, seeds, pks, BURST * (len(policies) * args.runs + 1), 2).reshape(-1, BURST, 128)
            want = eng.verify_rec128(votes.reshape(-1, 128)).reshape(-1, BURST)
            burst(q, votes[-1], want[-1])  # warm-up
            lat = {p: [] for p in policies}
            slices = {p: 0 for p in policies}
            k = 0
            for _ in range(args.runs):
                for p in policies:
                    done = threading.Event()
                    count = [0]

                    def loop(gap):
                        while not done.is_set():
                            one_slice()
                            count[0] += 1
                            if gap:
                                done.wait(gap)

                    th = None
                    if p != "none":
                        th = threading.Thread(target=loop, args=(PERIOD_S if p == "slice_every_15.6ms" else 0.0,))
                        th.start()
                    lat[p] += burst(q, votes[k], want[k])
                    k += 1
                    if th:
                        done.set()
                        th.join()
                    slices[p] += count[0]
            for p in policies:
                d = {"workload": "vote_burst_667x16_fresh", "policy": p, "runs": args.runs, "requests": len(lat[p]), "slice_buckets": SLICE,
                     "slices_run": slices[p]}
                d.update(stats_ms(lat[p]))
                emit(d)
        finally:
            q.close()
    finally:
        eng.close()
    if args.out:
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
