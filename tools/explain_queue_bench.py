#!/usr/bin/env python3
"""The verify queue's explain lane (hs_queue_submit_explain) against synchronous hs_explain_rec128 calls.

(a) Coalescing: K = 1, 16, 256 and 1,024 one-record explain requests of rejected records, submitted by 16 threads at once (K / 16 each),
    every thread then waiting for its own.  Time: host clock from the release of the threads to the last completion, median of --reps
    rounds after --warmup rounds.  The same K records as K synchronous Engine.explain calls from the same 16 threads.
(b) Votes under junk: a 667-vote burst (one-record requests from 16 threads, as tools/table_audit_bench.py) through one queue on a
    1,000-key committee, while one more thread explains one junk record at a time at a paced rate (0, 100, 400 and 1,600 per second, or
    as fast as the calls return), synchronously (Engine.explain: the context's mutex for the whole re-check) or through the lane
    (submit_explain; the thread does not wait).  Per vote: host clock from submit to verdict; the line holds the p50 and p99 over all
    votes of --reps bursts after one warm-up burst, and the explains completed during the bursts.
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/explain_queue_bench.py [--reps 7] [--warmup 2] [--out profiles/r02_explain_queue.jsonl]
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
KS = (1, 16, 256, 1024)
RATES = (0, 100, 400, 1600)
THREADS = 16


def smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unavailable"


def signed(eng, n_keys, n, seed):
    """n records signed on the GPU over n_keys keys (record i by key i % n_keys): (seeds, pks, records)."""
    rng = np.random.default_rng(seed)
    seeds = np.frombuffer(rng.bytes(32 * n_keys), np.uint8).reshape(n_keys, 32).copy()
    pks = eng.keygen_batch(seeds)
    ki = (np.arange(n) % n_keys).astype(np.uint32)
    digests = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    return seeds, pks, np.ascontiguousarray(np.concatenate([eng.sign_digests(seeds, pks, digests, ki), pks[ki], digests], axis=1))


def junk(recs, seed):
    """Each record with one seeded bit flipped anywhere in sig | pk | msg: rejected records."""
    out = recs.copy()
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 128 * 8, len(out))
    out[np.arange(len(out)), bits >> 3] ^= (1 << (bits & 7)).astype(np.uint8)
    return out


def run_threads(fn):
    go = threading.Barrier(THREADS + 1)
    th = [threading.Thread(target=lambda t=t: (go.wait(), fn(t))) for t in range(THREADS)]
    for x in th:
        x.start()
    go.wait()
    t0 = time.perf_counter()
    for x in th:
        x.join()
    return time.perf_counter() - t0


def coalescing(eng, q, recs, want, k, mode):
    out = np.zeros(k, np.uint8)

    def lane(t):
        mine = [(i, q.submit_explain(recs[i:i + 1])) for i in range(t, k, THREADS)]
        for i, tk in mine:
            out[i] = q.wait(tk)[0]

    def sync(t):
        for i in range(t, k, THREADS):
            out[i] = eng.explain(recs[i:i + 1])[0]
    dt = run_threads(lane if mode == "lane" else sync)
    assert (out == want[:k]).all(), "explain masks differ"
    return dt


def burst(q, votes, explain_one, rate):
    lat = np.zeros(len(votes))
    out = np.zeros(len(votes), bool)
    stop = threading.Event()
    done = [0]

    def explainer():
        period = 1.0 / rate if rate else 0.0
        nxt = time.perf_counter()
        i = 0
        while not stop.is_set():
            if explain_one(i):
                done[0] += 1
            i += 1
            nxt += period
            while period and not stop.is_set() and time.perf_counter() < nxt:
                time.sleep(min(1e-4, max(0.0, nxt - time.perf_counter())))

    def voter(t):
        for i in range(t, len(votes), THREADS):
            t0 = time.perf_counter()
            out[i] = q.wait(q.submit(votes[i:i + 1]))[0]
            lat[i] = time.perf_counter() - t0

    ex = threading.Thread(target=explainer) if explain_one else None
    if ex:
        ex.start()
        time.sleep(0.01)  # the junk is flowing when the burst starts
    run_threads(voter)
    stop.set()
    if ex:
        ex.join()
    return lat, out, done[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_explain_queue.jsonl"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("explain_queue_bench: no CUDA device (a time measured without the GPU means nothing)")
    from hotstuff_b200 import Engine
    card = smi()
    lines = []

    def emit(d):
        d["gpu"] = card
        lines.append(d)
        print(json.dumps(d), flush=True)

    eng = Engine(0)
    seeds, pks, valid = signed(eng, 1000, 4096, seed=7)
    bad = junk(valid, seed=8)
    want = eng.explain(bad)
    assert (want != 0).all(), "a flipped bit left a record valid"
    q = eng.queue()
    q.explain(1024, 1 << 20)

    # (a) K one-record requests from 16 threads: the lane against K synchronous calls
    for k in KS:
        for mode in ("sync", "lane"):
            for _ in range(a.warmup):
                coalescing(eng, q, bad, want, k, mode)
            st0 = q.explain_stats()
            ts = [coalescing(eng, q, bad, want, k, mode) for _ in range(a.reps)]
            st1 = q.explain_stats()
            med = statistics.median(ts)
            d = {"bench": "explain_coalescing", "mode": mode, "k": k, "threads": THREADS, "median_ms": round(med * 1e3, 3),
                 "min_ms": round(min(ts) * 1e3, 3), "max_ms": round(max(ts) * 1e3, 3), "reps": a.reps, "warmup": a.warmup,
                 "timing": "host clock from the threads' release to the last completion"}
            if mode == "lane":
                d["launches_per_round"] = round((st1["launches"] - st0["launches"]) / a.reps, 2)
            emit(d)

    # (b) a 667-vote burst on a 1,000-key committee with junk explains arriving, synchronous or through the lane
    assert eng.committee_register(pks).all()
    votes = valid[:667]
    for rate in RATES:
        for mode in (("none",) if rate == 0 else ("sync", "lane")):
            if mode == "sync":
                def explain_one(i):
                    return eng.explain(bad[i % len(bad):][:1]) is not None
            elif mode == "lane":
                def explain_one(i):
                    return q.submit_explain(bad[i % len(bad):][:1], callback=lambda *_: None) is not None
            else:
                explain_one = None
            burst(q, votes, explain_one, rate)  # warm-up
            lats, n_x, wall = [], 0, 0.0
            for _ in range(a.reps):
                t0 = time.perf_counter()
                lat, out, done = burst(q, votes, explain_one, rate)
                wall += time.perf_counter() - t0
                assert out.all(), "a valid vote was rejected"
                lats.append(lat)
                n_x += done
            lat = np.concatenate(lats)
            emit({"bench": "vote_burst_667x16_with_junk_explains", "committee_keys": 1000, "explain": mode, "target_rate_per_s": rate,
                  "explains_per_s": round(n_x / wall, 1), "vote_p50_us": round(float(np.percentile(lat, 50)) * 1e6, 1),
                  "vote_p99_us": round(float(np.percentile(lat, 99)) * 1e6, 1), "vote_max_us": round(float(lat.max()) * 1e6, 1),
                  "bursts": a.reps, "timing": "host clock from submit to verdict per vote"})
    q.explain(0, 0)  # waits for the lane's last requests
    emit({"bench": "explain_stats", **q.explain_stats()})
    q.close()
    eng.close()
    lines.append({"bench": "card_after", "gpu": smi()})
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
