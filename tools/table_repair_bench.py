#!/usr/bin/env python3
"""Cost of hs_table_repair (hotstuff_b200.Engine.table_repair), of the re-registration it replaces, and whether a repair in flight
moves a vote burst's latency.

The corrupt bytes come from the engine built with its test-only corruption hook (hs_test_poke, -DHS_TEST_HOOKS), which this tool
builds into a temporary directory unless --hook-lib names one.  One context: a committee of 4,096 keys from seeds at 13-bit key
windows (the window an 80 GB H100 picks for it), 24-bit base table.
  repair_slots_K  K = 1, 16, 256 slots with one comb-table entry flipped each, then one repair from the node's map: the first audit,
                  the slots taken out of service, rebuilt and proven, put back, and the final audit
  repair_base     one base-table entry flipped, then one repair: the base table rebuilt with the device drained, and the final audit
  register        hs_committee_register of the same 4,096 keys: the remedy the repair replaces (every table released and rebuilt)
  burst           667 single-vote requests from 16 threads through one verify queue, p50 of their submit-to-verdict latencies,
                  without and with a 64-slot repair in flight, alternated --reps times.  The flipped entries lie past any digit a
                  verify reads, so the votes' verdicts are exact throughout and are checked.
Time per call: host clock around the returning call (it ends in a stream synchronise), median of --reps.  Every line carries the card's
name, power limit and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/table_repair_bench.py [--reps 5] [--hook-lib PATH] [--out profiles/r02_table_repair.jsonl]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from table_audit_bench import burst, keys, ndigits, smi  # noqa: E402

ENTRY_BYTES = 96
POKE_TABLE, POKE_BASE = 0, 1
HS_AUDIT_TABLE, HS_AUDIT_BASE = 8, 16


def hook_lib(path):
    from hotstuff_b200 import _lib, build
    if not path:
        path = os.path.join(tempfile.mkdtemp(prefix="hs_hooks_"), "libhs_crypto_hooks.so")
        nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
        subprocess.check_call([nvcc] + build.NVCC_FLAGS + ["-DHS_TEST_HOOKS", "-o", path] +
                              [os.path.join(build.CSRC, f) for f in ("hs_engine.cu", "hs_ingest.cpp", "hs_multi.cpp")], cwd=build.ROOT)
    lib = ctypes.CDLL(path)
    for name, (res, args) in _lib.SIGNATURES.items():
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    lib.hs_test_poke.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint8]
    return lib


def engine(lib):
    from hotstuff_b200 import Engine
    h = ctypes.c_void_p()
    assert lib.hs_ctx_create(ctypes.byref(h), 0, 0) == 0 and h
    e = Engine._view(lib, h, 0)
    e._owned = True
    return e


def poke_unused(eng, slots):
    """One entry per slot in the top window, past any digit a canonical scalar gives, so verdicts stay exact until the repair."""
    W = eng.window_bits[0]
    top, H = ndigits(W) - 1, 1 << (W - 1)
    for k, s in enumerate(slots):
        off = ((top * (H + 1)) + H - (k % 64)) * ENTRY_BYTES + 7
        assert eng.lib.hs_test_poke(eng.h, POKE_TABLE, s, off, 0x10) == 0, eng.last_error


def timed_repair(eng, pks, want_found):
    t0 = time.perf_counter()
    found, failed, _ = eng.table_repair(pks)
    dt = time.perf_counter() - t0
    assert found == want_found and failed == 0, eng.last_error
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hook-lib", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_table_repair.jsonl"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("table_repair_bench: no GPU")
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
    rng = np.random.default_rng(1)
    timed_repair(eng, pks, 0)  # warm-up: the audit's stream and scratch
    for k in (1, 16, 256):
        ts = []
        for _ in range(args.reps):
            poke_unused(eng, sorted(rng.choice(4096, k, replace=False).tolist()))
            ts.append(timed_repair(eng, pks, HS_AUDIT_TABLE))
        emit(dict(workload="repair_slots_%d" % k, slots=k, repair_ms_median=round(statistics.median(ts) * 1e3, 3),
                  repair_ms_all=[round(t * 1e3, 3) for t in ts], **shape))
    ts = []
    stride = (1 << (wb - 1)) + 1
    for r in range(args.reps):
        assert lib.hs_test_poke(eng.h, POKE_BASE, (r % ndigits(wb)) * stride + 1 + r, 9, 0x10) == 0, eng.last_error
        ts.append(timed_repair(eng, pks, HS_AUDIT_BASE))
    emit(dict(workload="repair_base", repair_ms_median=round(statistics.median(ts) * 1e3, 3), repair_ms_all=[round(t * 1e3, 3) for t in ts],
              **shape))
    ts = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        eng.committee_register(pks)
        ts.append(time.perf_counter() - t0)
    emit(dict(workload="register", register_ms_median=round(statistics.median(ts) * 1e3, 3), register_ms_all=[round(t * 1e3, 3) for t in ts],
              **shape))
    # burst: 667 committee votes (a fifth of them with a flipped bit), judged by the oracle
    o = Oracle()
    ki = rng.integers(0, 4096, 667).astype(np.uint32)
    dig = np.frombuffer(rng.bytes(32 * 667), np.uint8).reshape(667, 32).copy()
    recs = np.zeros((667, 128), np.uint8)
    recs[:, :64], recs[:, 64:96], recs[:, 96:] = eng.sign_digests(seeds, pks, dig, key_idx=ki), pks[ki], dig
    recs[rng.random(667) < 0.2, 100] ^= 1
    want = o.verify_rec128(recs)
    q = eng.queue()
    burst(q, recs)  # warm-up
    p50 = {"without": [], "with": []}
    for _ in range(args.reps):
        t, got = burst(q, recs)
        assert np.array_equal(got, want)
        p50["without"].append(t)
        poke_unused(eng, sorted(set(ki[:64].tolist()) | set(rng.choice(4096, 64, replace=False).tolist()))[:64])
        res = {}
        th = threading.Thread(target=lambda: res.setdefault("r", eng.table_repair(pks)))
        th.start()
        t, got = burst(q, recs)
        th.join()
        assert np.array_equal(got, want) and res["r"][1] == 0, eng.last_error
        p50["with"].append(t)
    q.close()
    emit(dict(workload="burst", votes=667, threads=16, repair_slots=64,
              p50_ms_without=round(statistics.median(p50["without"]) * 1e3, 3), p50_ms_with=round(statistics.median(p50["with"]) * 1e3, 3),
              p50_ms_without_all=[round(t * 1e3, 3) for t in p50["without"]], p50_ms_with_all=[round(t * 1e3, 3) for t in p50["with"]],
              **shape))
    eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
