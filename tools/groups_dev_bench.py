#!/usr/bin/env python3
"""A stream of view-change bursts through the device-resident certificate pass against the host-pointer one, on one GPU.

Burst = N Timeouts (each its author's signature, strict, over the 16-byte Timeout preimage round || high_qc.round) plus ONE high_qc
(2N/3 + 1 votes, batch-eq, over its 40-byte preimage hash || round): N + 1 groups, the Timeouts' and the QC's.  64 bursts, each with
its own rounds and signatures, 1 % of the signatures corrupted.  The N Timeout authors are validators 0..N-1 of one registered
4,000-key committee, the QC's voters the first 2N/3 + 1 of them.

  (a) device: every burst's arrays resident in HBM; hs_verify_groups_dev + hs_qc_and_dev per burst on one stream with deferred mode
      on (the finish kernel and the AND of burst i run on the engine's tail stream beside burst i + 1), closed by ONE hs_results_wait;
      CUDA events around the 64 bursts.
  (b) host: the same 64 bursts through 64 hs_verify_groups calls (host arrays; copies, pass, copy back, synchronise), host clock.

Every group and item bit of (a) is checked against (b) before anything is timed.  Prints one JSON line per N with the card's name and
power limit read in the same run, plus the median, min and max over the repetitions.

    python tools/groups_dev_bench.py [--n 100,1000,4000] [--reps 7] [--bursts 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
COMMITTEE = 4000


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q or "unavailable"}


def make_bursts(eng, seeds, pks, n, n_bursts, rng):
    """Host arrays of n_bursts view-change bursts of n Timeouts each (see the module docstring)."""
    q = 2 * n // 3 + 1
    items = n + q
    out = []
    for b in range(n_bursts):
        rnd = 1000 + 10 * b
        pre = bytearray()
        for i in range(n):
            pre += (rnd + i % 3).to_bytes(8, "little") + (rnd - 1).to_bytes(8, "little")  # Timeout: round || high_qc.round
        pre += rng.bytes(32) + (rnd - 1).to_bytes(8, "little")                           # high_qc: hash || round
        pre = np.frombuffer(bytes(pre), np.uint8).copy()
        off = np.concatenate([np.arange(n + 1, dtype=np.uint64) * 16, [n * 16 + 40]]).astype(np.uint64)
        mi = np.concatenate([np.arange(n), np.full(q, n)]).astype(np.uint32)
        gi = mi.copy()  # group i = Timeout i, group n = the high_qc
        modes = np.concatenate([np.zeros(n), np.ones(q)]).astype(np.uint8)
        kidx = np.concatenate([np.arange(n), np.arange(q)]).astype(np.uint32)
        dig = eng.digest32_batch(pre, off)
        sig = eng.sign_digests(seeds, pks, dig[mi], key_idx=kidx)
        bad = np.flatnonzero(rng.random(items) < 0.01)
        sig[bad, rng.integers(0, 64, bad.size)] ^= (1 << rng.integers(0, 8, bad.size)).astype(np.uint8)
        out.append(dict(pre=pre, off=off, sig=sig, pk=pks[kidx].copy(), mi=mi, gi=gi, modes=modes, n_groups=n + 1, n_items=items))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="100,1000,4000")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--bursts", type=int, default=64)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("groups_dev_bench: needs a CUDA device")
    from hotstuff_b200 import Engine
    from hotstuff_b200.engine import bitmap_to_bools
    info = card()
    rng = np.random.default_rng(2024)
    eng = Engine(0)
    seeds = rng.integers(0, 256, (COMMITTEE, 32), dtype=np.uint8)
    pks = eng.keygen_batch(seeds)
    assert eng.committee_register(pks).all()
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    for n in [int(x) for x in args.n.split(",")]:
        bursts = make_bursts(eng, seeds, pks, n, args.bursts, rng)
        d = [dict(pre=t(b["pre"]), off=t(b["off"].view(np.int64)), sig=t(b["sig"]), pk=t(b["pk"]), mi=t(b["mi"].view(np.int32)), gi=t(b["gi"].view(np.int32)),
                  mode=t(b["modes"]), ib=torch.zeros((b["n_items"] + 31) // 32, dtype=torch.int32, device=dev),
                  gb=torch.zeros((b["n_groups"] + 31) // 32, dtype=torch.int32, device=dev)) for b in bursts]

        def host_stream():
            return [eng.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], b["n_groups"], mode=b["modes"], pk=b["pk"], want_items=True)
                    for b in bursts]

        def dev_stream():
            for b, x in zip(bursts, d):
                eng.verify_groups_dev(x["pre"], x["off"], len(b["off"]) - 1, x["sig"], x["mi"], x["ib"], b["n_items"], d_mode=x["mode"], d_pk=x["pk"])
                eng.qc_and_dev(x["ib"], x["gi"], b["n_items"], b["n_groups"], x["gb"])
            eng.results_wait()

        want = host_stream()
        eng.set_deferred(True)
        for x in d:
            x["ib"].fill_(-1)
            x["gb"].fill_(-1)
        dev_stream()
        torch.cuda.synchronize()
        for b, x, (wg, wi) in zip(bursts, d, want):
            assert (bitmap_to_bools(x["ib"].cpu().numpy().view(np.uint32), b["n_items"]) == wi).all(), "item bits differ from hs_verify_groups"
            assert (bitmap_to_bools(x["gb"].cpu().numpy().view(np.uint32), b["n_groups"]) == wg).all(), "group bits differ from hs_verify_groups"
        rejected = int(sum((~wi).sum() for _, wi in want))
        assert rejected > 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dev_ms, host_ms = [], []
        for _ in range(args.reps):  # the two arms alternate, so drift on a shared host hits both
            eng.set_deferred(True)
            torch.cuda.synchronize()
            e0.record()
            dev_stream()
            e1.record()
            torch.cuda.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
            eng.set_deferred(False)
            t0 = time.perf_counter()
            host_stream()
            host_ms.append((time.perf_counter() - t0) * 1e3)
        stat = lambda v: {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)}
        print(json.dumps(dict(info, n_timeouts=n, qc_votes=2 * n // 3 + 1, bursts=args.bursts, items_per_burst=bursts[0]["n_items"], reps=args.reps,
                              rejected_items=rejected, device_deferred_ms=stat(dev_ms), host_calls_ms=stat(host_ms),
                              speedup_median=round(float(np.median(host_ms) / np.median(dev_ms)), 3))), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
