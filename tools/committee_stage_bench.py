#!/usr/bin/env python3
"""Cost of a committee change made at once (hs_committee_update) against one staged off the verify path and switched in with a commit
(hs_committee_stage + hs_committee_commit), and what each does to a vote burst's latency.

One context: a committee of 4,096 keys from seeds at the default key window (13 bits on an 80 GB H100), 24-bit base table.  Every
change adds K new keys and removes K live validators, K = 16 and 256.
  change_K   wall time of update(A, R), and of stage(A, R) and commit(), alternated --reps times (a host clock around each returning
             call).  The stage is what a node runs in the last rounds of an epoch; the commit is what stops the votes at the boundary.
  burst_K    667 single-vote requests from 16 threads through one verify queue: per-vote submit-to-verdict latency p50, p99 and max over
             --reps bursts per arm, for three arms alternated: the burst alone, with the update started as the burst starts, and with
             the stage started as the burst starts and the commit right after it.  Verdicts are checked against the oracle.
  audit_full hs_table_audit of the whole committee after the changes, median of --reps.
  repair_256 hs_table_repair of 256 slots with one comb-table entry flipped each, through the engine built with its test-only
             corruption hook (hs_test_poke, -DHS_TEST_HOOKS; built into a temporary directory unless --hook-lib names one).
Every line carries the card's name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/committee_stage_bench.py [--reps 5] [--hook-lib PATH] [--out profiles/r02_committee_stage.jsonl]
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
from table_audit_bench import keys, smi, time_audit  # noqa: E402
from table_repair_bench import HS_AUDIT_TABLE, engine, hook_lib, poke_unused, timed_repair  # noqa: E402


def burst(q, recs, threads=16):
    """Every vote's submit-to-verdict latency (seconds) and the verdicts."""
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
    return lat, np.array(out, bool)


def ms(x):
    return round(x * 1e3, 3)


def summary(lats):
    a = np.array(lats)
    return {"p50_ms": ms(float(np.percentile(a, 50))), "p99_ms": ms(float(np.percentile(a, 99))), "max_ms": ms(float(a.max()))}


class Committee:
    """The engine's committee and the node's map; fresh keys come from a pool of seeded keys."""

    def __init__(self, eng, pool):
        self.eng, self.pool, self.next = eng, pool, 4096
        self.key = {s: s for s in range(4096)}  # slot in service -> index of its key in the pool

    def change(self, k, rng):
        """K fresh keys (pool indices) and K live slots to remove."""
        add = np.arange(self.next, self.next + k)
        self.next += k
        rem = sorted(rng.choice(sorted(self.key), k, replace=False).tolist())
        return add, np.array(rem, np.uint32)

    def _applied(self, add, idx, rem):
        for s in rem.tolist():
            del self.key[s]
        self.key.update({int(i): int(a) for i, a in zip(idx, add)})

    def update(self, add, rem):
        t0 = time.perf_counter()
        idx = self.eng.committee_update(self.pool[add], rem)
        dt = time.perf_counter() - t0
        # one update removes first, so an added key may take a slot it frees
        for s in rem.tolist():
            del self.key[s]
        self._applied(add, idx, np.zeros(0, np.uint32))
        return dt

    def stage_commit(self, add, rem):
        t0 = time.perf_counter()
        idx = self.eng.committee_stage(self.pool[add], rem)
        t1 = time.perf_counter()
        self.eng.committee_commit()
        t2 = time.perf_counter()
        self._applied(add, idx, rem)
        return t1 - t0, t2 - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hook-lib", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_committee_stage.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("committee_stage_bench: no GPU")
    from hotstuff_b200 import Engine
    from oracle_api import Oracle
    card = smi()
    lines = []

    def emit(d):
        d["card"] = card
        print(json.dumps(d), flush=True)
        lines.append(d)

    o = Oracle()
    eng = Engine(0)
    n_pool = 4096 + 2 * args.reps * 3 * (16 + 256) + 512
    seeds, pool = keys(eng, n_pool, 4096)
    eng.committee_register(pool[:4096])
    wa, wb = eng.window_bits
    shape = {"committee_keys": 4096, "key_slots": eng.key_slots, "key_window": wa, "base_window": wb}
    C = Committee(eng, pool)
    rng = np.random.default_rng(1)
    # warm-up: the audit's stream and scratch, the staging buffers, the verify queue
    C.update(*C.change(16, rng))
    C.stage_commit(*C.change(16, rng))
    for k in (16, 256):
        up, st, cm = [], [], []
        for _ in range(args.reps):
            up.append(C.update(*C.change(k, rng)))
            s, c = C.stage_commit(*C.change(k, rng))
            st.append(s)
            cm.append(c)
        emit(dict(workload="change_%d" % k, added=k, removed=k, update_ms_median=ms(statistics.median(up)),
                  stage_ms_median=ms(statistics.median(st)), commit_ms_median=ms(statistics.median(cm)), update_ms_all=[ms(t) for t in up],
                  stage_ms_all=[ms(t) for t in st], commit_ms_all=[ms(t) for t in cm], **shape))
    med, ts = time_audit(eng, args.reps)  # the full audit runs the list-capable k_table_audit without a list
    emit(dict(workload="audit_full", audit_ms_median=ms(med), audit_ms_all=[ms(t) for t in ts], **dict(shape, key_slots=eng.key_slots)))
    q = eng.queue()
    for k in (16, 256):
        lat = {"alone": [], "update": [], "stage_commit": []}
        for _ in range(args.reps):
            for arm in ("alone", "update", "stage_commit"):
                recs = votes(eng, seeds, C, rng)
                want = o.verify_rec128(recs)
                th = None
                if arm != "alone":
                    change = C.change(k, rng)
                    fn = C.update if arm == "update" else C.stage_commit
                    th = threading.Thread(target=fn, args=change)
                    th.start()
                t, got = burst(q, recs)
                if th:
                    th.join()
                assert np.array_equal(got, want)
                lat[arm].extend(t)
        d = dict(workload="burst_%d" % k, votes=667, threads=16, added=k, removed=k, bursts_per_arm=args.reps)
        for arm, v in lat.items():
            d.update({"%s_%s" % (arm, key): val for key, val in summary(v).items()})
        emit(dict(d, **shape))
    q.close()
    eng.close()
    # repair of 256 slots, as in tools/table_repair_bench.py
    lib = hook_lib(args.hook_lib)
    h = engine(lib)
    hseeds, hpks = keys(h, 4096, 4096)
    h.committee_register(hpks)
    timed_repair(h, hpks, 0)
    ts = []
    for _ in range(args.reps):
        poke_unused(h, sorted(rng.choice(4096, 256, replace=False).tolist()))
        ts.append(timed_repair(h, hpks, HS_AUDIT_TABLE))
    emit(dict(workload="repair_256", slots=256, repair_ms_median=ms(statistics.median(ts)), repair_ms_all=[ms(t) for t in ts],
              key_slots=h.key_slots, key_window=h.window_bits[0], base_window=h.window_bits[1]))
    h.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")


def votes(eng, seeds, C, rng, n=667):
    """n votes over one Digest by validators in service, a fifth of them with a flipped bit."""
    ki = np.array([C.key[s] for s in rng.choice(sorted(C.key), n, replace=False)], np.uint32)
    dig = np.frombuffer(rng.bytes(32), np.uint8)
    sig = eng.sign_digests(seeds, C.pool, np.tile(dig, (n, 1)), key_idx=ki)
    recs = np.concatenate([sig, C.pool[ki], np.tile(dig, (n, 1))], axis=1)
    recs[rng.random(n) < 0.2, 100] ^= 1
    return recs


if __name__ == "__main__":
    main()
