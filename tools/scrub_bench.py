#!/usr/bin/env python3
"""What the engine-owned scrub (hs_scrub_start) costs a tick, and what it and a periodic full audit do to a vote burst's latency.

One context: a 4,096-key committee at 13-bit key windows and the 24-bit base-point table (8.9 GB), registered as a node would.
Tick cost: the scrub with a 1 us period (ticks back to back), from its own counters over 1 s of wall time: the host clock per tick,
which ends in a stream synchronise, so it bounds the tick's GPU time from above.  A pass's slot part and base part each idle once done
until the other is, so each run keeps both busy: base slices alone on a context without per-key tables (a least-squares line gives the
cost per million base entries), then the committee at K ticks per pass (4096 / K slots and E / K base entries a tick); less the base
part, a line in the slots gives the cost per slot, and its intercept a tick's fixed cost (the slot checks of every slot and hash entry,
the launches and the synchronises).
Burst: 667 single-vote requests from 16 threads through one verify queue, repeated back to back for --window seconds under each
policy, alternated --reps times; p50, p99 and max of every request's submit-to-verdict latency, verdicts checked against the engine's
quiet answers.  Policies: (a) nothing; (b) a full hs_table_audit every --period seconds from another thread; (c) the scrub at
ticks-per-pass K, with period --period / K, so a pass takes the same --period.
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/scrub_bench.py [--reps 3] [--window 3] [--period 0.5] [--out profiles/r02_scrub.jsonl]
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
from table_audit_bench import entries, keys, smi  # noqa: E402

N_KEYS, KEY_WINDOW = 4096, 13
TICKS_PER_PASS = (8, 32, 128)


def tick_cost(eng, pks, slots, base, window):
    """Seconds per tick and ticks run, the scrub running back to back for `window` seconds."""
    eng.scrub_start(pks, None, period_us=1, slots_per_tick=slots, base_entries_per_tick=base)
    try:
        time.sleep(0.2)  # warm-up ticks
        t0, s0 = time.perf_counter(), eng.scrub_stats()
        time.sleep(window)
        t1, s1 = time.perf_counter(), eng.scrub_stats()
    finally:
        eng.scrub_stop()
    ticks = s1["ticks"] - s0["ticks"]
    assert ticks > 0 and s1["findings"] == 0, s1
    return (t1 - t0) / ticks, ticks


def fit(xs, ys):
    a, b = np.polyfit(np.asarray(xs, float), np.asarray(ys, float), 1)
    return float(a), float(b)


def votes(eng, seeds, pks, n=667, seed=7):
    rng = np.random.default_rng(seed)
    ki = rng.integers(0, len(pks), n).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32).copy()
    recs = np.zeros((n, 128), np.uint8)
    recs[:, :64] = eng.sign_digests(seeds, pks, dig, key_idx=ki)
    recs[:, 64:96] = pks[ki]
    recs[:, 96:] = dig
    return recs


def bursts(q, recs, want, window, threads=16):
    """Bursts back to back for `window` seconds: every request's latency (seconds) and the number of bursts."""
    lat, n_bursts = [], 0
    end = time.perf_counter() + window
    while time.perf_counter() < end:
        one = [0.0] * len(recs)
        out = [None] * len(recs)

        def worker(t):
            for i in range(t, len(recs), threads):
                t0 = time.perf_counter()
                out[i] = q.wait(q.submit(recs[i:i + 1]))[0]
                one[i] = time.perf_counter() - t0

        th = [threading.Thread(target=worker, args=(t,)) for t in range(threads)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert np.array_equal(np.array(out, bool), want)
        lat += one
        n_bursts += 1
    return lat, n_bursts


def stats_ms(lat):
    a = np.asarray(lat) * 1e3
    return {"p50_ms": round(float(np.percentile(a, 50)), 4), "p99_ms": round(float(np.percentile(a, 99)), 4), "max_ms": round(float(a.max()), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=3.0)
    ap.add_argument("--period", type=float, default=0.5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_scrub.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("scrub_bench: no GPU")
    from hotstuff_b200 import Engine
    card = smi()
    lines = []

    def emit(d):
        d["card"] = card
        print(json.dumps(d), flush=True)
        lines.append(d)

    base_only = Engine(0)
    try:
        base_pts = [(b, tick_cost(base_only, None, 1, b, 1.0)) for b in (1 << 18, 1 << 20, 1 << 22, 1 << 24)]
    finally:
        base_only.close()
    per_entry, fixed_b = fit([b for b, _ in base_pts], [t for _, (t, _) in base_pts])
    eng = Engine(0, key_window=KEY_WINDOW)
    try:
        seeds, pks = keys(eng, N_KEYS, N_KEYS)
        eng.committee_register(pks)
        wa, wb = eng.window_bits
        E = entries(wb)
        t0 = time.perf_counter()
        assert eng.table_audit(pks)[0] == 0, eng.last_error
        full_ms = (time.perf_counter() - t0) * 1e3
        pts = [(-(-N_KEYS // k), -(-E // k), tick_cost(eng, pks, -(-N_KEYS // k), -(-E // k), 1.0)) for k in (8, 32, 128, 512)]
        per_slot, fixed_s = fit([s for s, _, _ in pts], [t - b * per_entry for _, b, (t, _) in pts])
        emit({"workload": "tick_cost", "key_slots": N_KEYS, "key_window": wa, "base_window": wb, "base_entries": E,
              "full_audit_ms_once": round(full_ms, 3),
              "base_only_ticks": [{"base_entries_per_tick": b, "tick_ms": round(t * 1e3, 4), "ticks": n} for b, (t, n) in base_pts],
              "committee_ticks": [{"slots_per_tick": s, "base_entries_per_tick": b, "tick_ms": round(t * 1e3, 4), "ticks": n}
                                  for s, b, (t, n) in pts],
              "ms_per_million_base_entries": round(per_entry * 1e9, 4), "tick_fixed_ms_base_only": round(fixed_b * 1e3, 4),
              "us_per_slot": round(per_slot * 1e6, 3), "tick_fixed_ms_committee": round(fixed_s * 1e3, 4)})

        recs = votes(eng, seeds, pks)
        want = eng.verify_rec128(recs)
        q = eng.queue()
        try:
            bursts(q, recs, want, 0.5)  # warm-up
            runs = {"none": [], "full_audit": []}
            runs.update({"scrub_k%d" % k: [] for k in TICKS_PER_PASS})
            work = {name: [] for name in runs}
            for _ in range(args.reps):
                for name in runs:
                    done = threading.Event()
                    count = [0]
                    if name == "full_audit":
                        def loop():
                            while not done.is_set():
                                t = time.perf_counter()
                                assert eng.table_audit(pks)[0] == 0
                                count[0] += 1
                                done.wait(max(0.0, args.period - (time.perf_counter() - t)))
                        th = threading.Thread(target=loop)
                        th.start()
                    elif name.startswith("scrub"):
                        k = int(name[len("scrub_k"):])
                        eng.scrub_start(pks, None, period_us=int(args.period * 1e6 / k), slots_per_tick=-(-N_KEYS // k),
                                        base_entries_per_tick=-(-E // k))
                        s0 = eng.scrub_stats()["passes"]
                    lat, nb = bursts(q, recs, want, args.window)
                    if name == "full_audit":
                        done.set()
                        th.join()
                        work[name].append(count[0])
                    elif name.startswith("scrub"):
                        st = eng.scrub_stats()
                        eng.scrub_stop()
                        assert st["findings"] == 0, st
                        work[name].append(st["passes"] - s0)
                    runs[name] += lat
            for name, lat in runs.items():
                d = {"workload": "vote_burst_667x16", "policy": name, "period_s": args.period, "window_s": args.window, "reps": args.reps,
                     "requests": len(lat)}
                d.update(stats_ms(lat))
                if name == "full_audit":
                    d["audits_per_window"] = work[name]
                elif name.startswith("scrub"):
                    k = int(name[len("scrub_k"):])
                    d.update({"ticks_per_pass": k, "period_us": int(args.period * 1e6 / k), "slots_per_tick": -(-N_KEYS // k),
                              "base_entries_per_tick": -(-E // k), "passes_per_window": work[name]})
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
