#!/usr/bin/env python3
"""Cost of hs_table_mend (hotstuff_b200.Engine.table_mend) against hs_table_repair for the same finding, and what each does to a vote
burst in flight beside it.

The corrupt bytes come from the engine built with its test-only corruption hook (hs_test_poke, -DHS_TEST_HOOKS), built into a temporary
directory unless --hook-lib names one.  One context: a committee of 4,096 keys from seeds at 13-bit key windows (the window an 80 GB
H100 picks for it), 24-bit base table.  Every flipped entry lies past any digit a verify reads (the top window's high entries), so
verdicts are exact throughout and are checked against the oracle.
  base_entry   one base-table entry flipped, then one mend (its locating audit, the window recomputed, the proof) or one repair (the
               whole base table rebuilt with the device drained, and the final audit), alternated --reps times
  slot_entry   one comb-table entry of one slot flipped, then one mend or one repair (the slot out of service, rebuilt and proven),
               alternated --reps times
  burst        667 single-vote requests from 16 threads through one verify queue, p50 and p99 of their submit-to-verdict latencies:
               without anything beside them, beside a base mend, beside a base repair, alternated --reps times
Time per call: host clock around the returning call (it ends in a stream synchronise), median of --reps.  Every line carries the card's
name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/table_mend_bench.py [--reps 5] [--hook-lib PATH] [--out profiles/r02_table_mend.jsonl]
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
from table_audit_bench import keys, ndigits, smi  # noqa: E402
from table_repair_bench import engine, hook_lib  # noqa: E402

ENTRY_BYTES = 96
POKE_TABLE, POKE_BASE = 0, 1
HS_AUDIT_TABLE, HS_AUDIT_BASE = 8, 16


def burst(q, recs, threads=16):
    """Latencies (s) and verdicts of len(recs) single-vote requests from `threads` threads."""
    lat, out = [0.0] * len(recs), [None] * len(recs)

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


def ms(v):
    return round(v * 1e3, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hook-lib", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_table_mend.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("table_mend_bench: no GPU")
    from oracle_api import Oracle
    lib = hook_lib(args.hook_lib)
    card = smi()
    lines = []

    def emit(d):
        d["card"] = card
        print(json.dumps(d), flush=True)
        lines.append(d)

    eng = engine(lib)
    seeds, pks = keys(eng, 4096, 4096)
    eng.committee_register(pks)
    wa, wb = eng.window_bits
    shape = {"key_slots": eng.key_slots, "key_window": wa, "base_window": wb}
    rng = np.random.default_rng(2)
    btop, bH = ndigits(wb) - 1, 1 << (wb - 1)
    ktop, kH = ndigits(wa) - 1, 1 << (wa - 1)

    def poke_base(k):
        assert lib.hs_test_poke(eng.h, POKE_BASE, btop * (bH + 1) + bH - k, 9, 0x10) == 0, eng.last_error

    def poke_slot(s, k):
        assert lib.hs_test_poke(eng.h, POKE_TABLE, s, (ktop * (kH + 1) + kH - k) * ENTRY_BYTES + 7, 0x10) == 0, eng.last_error

    def timed(fn, want):
        t0 = time.perf_counter()
        r = fn(pks)
        dt = time.perf_counter() - t0
        assert r[0] == want and r[1] == 0, eng.last_error
        return dt

    eng.table_mend(pks)  # warm-up: the audit's stream and scratch
    poke_base(0)
    timed(eng.table_mend, HS_AUDIT_BASE)  # and the mend's staging
    for name, poke, want in (("base_entry", poke_base, HS_AUDIT_BASE), ("slot_entry", None, HS_AUDIT_TABLE)):
        t = {"mend": [], "repair": []}
        for r in range(args.reps):
            for how, fn in (("mend", eng.table_mend), ("repair", eng.table_repair)):
                if poke:
                    poke(r + 1)
                else:
                    poke_slot(int(rng.integers(0, 4096)), r + 1)
                t[how].append(timed(fn, want))
        emit(dict(workload=name, mend_ms_median=ms(statistics.median(t["mend"])), repair_ms_median=ms(statistics.median(t["repair"])),
                  mend_ms_all=[ms(x) for x in t["mend"]], repair_ms_all=[ms(x) for x in t["repair"]], **shape))
    o = Oracle()
    ki = rng.integers(0, 4096, 667).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * 667), np.uint8).reshape(667, 32).copy()
    recs = np.zeros((667, 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = eng.sign_digests(seeds, pks, dig, key_idx=ki), pks[ki], dig
    recs[rng.random(667) < 0.2, 100] ^= 1
    want = o.verify_rec128(recs)
    q = eng.queue()
    burst(q, recs)  # warm-up
    lat = {"alone": [], "mend": [], "repair": []}
    for r in range(args.reps):
        for how in ("alone", "mend", "repair"):
            res, th = {}, None
            if how != "alone":
                poke_base(10 + r)
                fn = eng.table_mend if how == "mend" else eng.table_repair
                th = threading.Thread(target=lambda: res.setdefault("r", fn(pks)))
                th.start()
                time.sleep(0.07)  # past the locating audit (about 69 ms): the burst meets the mend's stores or the repair's rebuild
            l, got = burst(q, recs)
            if th:
                th.join()
                assert res["r"][1] == 0, eng.last_error
            assert np.array_equal(got, want)
            lat[how].append(l)
    q.close()
    d = dict(workload="burst", votes=667, threads=16, **shape)
    for how, runs in lat.items():
        d["p50_ms_" + how] = ms(statistics.median(statistics.median(l) for l in runs))
        d["p99_ms_" + how] = ms(statistics.median(float(np.percentile(l, 99)) for l in runs))
        d["p99_ms_%s_all" % how] = [ms(float(np.percentile(l, 99))) for l in runs]
    emit(d)
    st = eng.mend_stats()
    emit(dict(workload="mend_stats", **st, **shape))
    eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
