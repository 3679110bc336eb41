#!/usr/bin/env python3
"""Cost of a whole re-registration made at once (hs_committee_register) against one staged beside the live store and switched in with a
commit (hs_committee_stage_register + hs_committee_commit), and what each does to a vote burst's latency.

One context per committee size N = 1,024 and 4,096 (keys from seeds), registered at the default key window, 24-bit base table.  Every
change re-registers the same N keys, so the votes stay valid across it.
  change_N   wall time of register(P), and of stage_register(P) and commit(), alternated --reps times (a host clock around each returning
             call).  The stage takes the widest window that fits beside the live store (key_bits 0), reported as stage_window.  The commit
             includes the free of the old store after the context's mutex is released; discard_ms is hs_committee_discard of a staged
             store of the same size, i.e. that free alone, so commit_ms - discard_ms is the drain and the swap.
  burst_N    667 single-vote requests from 16 threads through one verify queue: per-vote submit-to-verdict latency p50, p99 and max over
             --reps bursts per arm, for four arms alternated: the burst alone; the registration started as the burst starts; the stage
             started as the burst starts (then discarded); and the commit of a stage built before the burst, called once a quarter of
             the votes have returned, so that it lands in the burst's middle.  For each change arm, the same statistics over the votes in
             flight at some point of the change's call (submitted before it returned, returned after it started).  Verdicts are checked
             against the oracle.
  burst_N_timeline  per burst: its length, and the change's start and end, the votes in flight during it, the votes that had
             returned before it started and those submitted after it ended (ms from the burst's start, host clock).
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/committee_stage_register_bench.py [--reps 5] [--out profiles/r02_committee_stage_register.jsonl]
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from committee_stage_bench import ms, summary  # noqa: E402
from table_audit_bench import keys, smi  # noqa: E402


def timed_burst(q, recs, trigger, after, threads=16):
    """Every vote's submit and return time (host clock, seconds) and the verdicts; `trigger` is set once `after` votes have returned."""
    sub = np.zeros(len(recs))
    ret = np.zeros(len(recs))
    out = [None] * len(recs)
    done = [0]
    lock = threading.Lock()

    def worker(t):
        for i in range(t, len(recs), threads):
            sub[i] = time.perf_counter()
            out[i] = q.wait(q.submit(recs[i:i + 1]))[0]
            ret[i] = time.perf_counter()
            with lock:
                done[0] += 1
                if done[0] == after:
                    trigger.set()

    th = [threading.Thread(target=worker, args=(t,)) for t in range(threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return sub, ret, np.array(out, bool)


def timed(fn, *a):
    t0 = time.perf_counter()
    r = fn(*a)
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1024,4096")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_committee_stage_register.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("committee_stage_register_bench: no GPU")
    from hotstuff_b200 import Engine
    from oracle_api import Oracle
    card = smi()
    lines = []

    def emit(d):
        d["card"] = card
        print(json.dumps(d), flush=True)
        lines.append(d)

    o = Oracle()
    rng = np.random.default_rng(2)
    for n in [int(x) for x in args.sizes.split(",")]:
        eng = Engine(0)
        seeds, pks = keys(eng, n, n)
        eng.committee_register(pks)
        wa, wb = eng.window_bits
        shape = {"committee_keys": n, "key_slots": eng.key_slots, "key_window": wa, "base_window": wb}

        def stage_commit():
            ts, (_, bits) = timed(eng.committee_stage_register, pks)
            tc, _ = timed(eng.committee_commit)
            return ts, tc, bits

        # warm-up: the audit's stream and scratch, the allocator, the verify queue
        stage_commit()
        eng.committee_register(pks)
        reg, st, cm, dc, windows = [], [], [], [], set()
        for _ in range(args.reps):
            reg.append(timed(eng.committee_register, pks)[0])
            s, c, bits = stage_commit()
            st.append(s)
            cm.append(c)
            windows.add(bits)
            eng.committee_stage_register(pks)
            dc.append(timed(eng.committee_discard)[0])
        assert len(windows) == 1
        emit(dict(workload="change_%d" % n, stage_window=windows.pop(), register_ms_median=ms(statistics.median(reg)),
                  stage_ms_median=ms(statistics.median(st)), commit_ms_median=ms(statistics.median(cm)),
                  discard_ms_median=ms(statistics.median(dc)), register_ms_all=[ms(t) for t in reg], stage_ms_all=[ms(t) for t in st],
                  commit_ms_all=[ms(t) for t in cm], discard_ms_all=[ms(t) for t in dc], **shape))
        eng.committee_register(pks)  # back to the registration's window for the bursts
        q = eng.queue()
        arms = ("alone", "register", "stage", "commit")
        lat = {a: [] for a in arms}
        inside = {a: [] for a in arms}  # latencies of the votes in flight at some point of the change's call
        timelines = []
        for rep in range(args.reps):
            for arm in arms:
                ki = rng.choice(n, 667, replace=n < 667).astype(np.uint32)
                dig = np.frombuffer(rng.bytes(32), np.uint8)
                sig = eng.sign_digests(seeds, pks, np.tile(dig, (667, 1)), key_idx=ki)
                recs = np.concatenate([sig, pks[ki], np.tile(dig, (667, 1))], axis=1)
                recs[rng.random(667) < 0.2, 100] ^= 1
                want = o.verify_rec128(recs)
                if arm == "commit":
                    eng.committee_stage_register(pks)  # built before the burst: only the commit meets it
                trigger = threading.Event()
                span = {}

                def change(arm=arm, trigger=trigger, span=span):
                    if arm == "commit":
                        trigger.wait()  # a quarter of the votes have returned: the burst is in full flow
                    span["start"] = time.perf_counter()
                    if arm == "register":
                        eng.committee_register(pks)
                    elif arm == "stage":
                        eng.committee_stage_register(pks)
                    else:
                        eng.committee_commit()
                    span["end"] = time.perf_counter()

                th = None if arm == "alone" else threading.Thread(target=change)
                t0 = time.perf_counter()
                if th:
                    th.start()
                sub, ret, got = timed_burst(q, recs, trigger, len(recs) // 4)
                if th:
                    th.join()
                else:
                    trigger.set()
                if arm == "stage":
                    eng.committee_discard()
                elif arm == "commit" and eng.window_bits[0] != wa:
                    eng.committee_register(pks)  # the next arms start from the registration's window
                assert np.array_equal(got, want)
                lat[arm].extend((ret - sub).tolist())
                tl = dict(rep=rep, arm=arm, burst_ms=ms(float(ret.max() - t0)))
                if th:
                    a, b = span["start"], span["end"]
                    hit = (sub < b) & (ret > a)
                    inside[arm].extend((ret - sub)[hit].tolist())
                    tl.update(change_start_ms=ms(a - t0), change_end_ms=ms(b - t0), votes_in_flight_during_change=int(hit.sum()),
                              votes_returned_before_change=int((ret <= a).sum()), votes_submitted_after_change=int((sub >= b).sum()))
                timelines.append(tl)
        q.close()
        d = dict(workload="burst_%d" % n, votes=667, threads=16, bursts_per_arm=args.reps, commit_after_votes=667 // 4)
        for arm in arms:
            d.update({"%s_%s" % (arm, key): val for key, val in summary(lat[arm]).items()})
            if inside[arm]:
                d.update({"%s_overlapping_%s" % (arm, key): val for key, val in summary(inside[arm]).items()})
                d["%s_overlapping_votes" % arm] = len(inside[arm])
        emit(dict(d, **shape))
        emit(dict(workload="burst_%d_timeline" % n, bursts=timelines, **shape))
        eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
