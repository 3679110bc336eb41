#!/usr/bin/env python3
"""Cost of hs_explain_groups_dev after a 2^20-item hs_verify_groups_dev pass, and what an explanation flood costs verify passes beside it.

Workload: 2^20 items signed on the GPU by 1,024 registered keys (key bytes), over 4,096 QC-shaped 40-byte preimages, every other item
batch-eq.  For r = 0, 1, 64, 4,096 and 65,536 rejected items (a bit flipped in R of r items), the pass runs once and its item bitmap is
checked (exactly r zero bits); then the explanation is timed with CUDA events on the same stream at max_explain = 0 (every rejected
item) and 64, and its out words are checked (r zero bits, min(r, cap) examined, no engine fault).

Interference: a stream of 4,096-item groups_dev passes on a second stream, each timed with CUDA events, alone and with a 65,536-item
explanation enqueued just before on a third stream; the two arms alternate.  Prints one JSON line per measurement with the card's name
and power limit read in the same run.

    python tools/explain_dev_bench.py [--reps 10] [--rounds 8] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N_ITEMS, N_KEYS, N_MSGS = 1 << 20, 1024, 4096
REJECTED = (0, 1, 64, 4096, 65536)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q or "unavailable", "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def stats(ms):
    ms = np.asarray(ms)
    return {"p50_ms": round(float(np.median(ms)), 4), "p99_ms": round(float(np.percentile(ms, 99)), 4), "min_ms": round(float(ms.min()), 4),
            "max_ms": round(float(ms.max()), 4), "n": int(ms.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--passes", type=int, default=24, help="4,096-item passes per interference round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("explain_dev_bench: needs a CUDA device")
    from hotstuff_b200 import Engine
    info = card()
    lines = []

    def emit(d):
        d.update(info)
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))

    rng = np.random.default_rng(7)
    eng = Engine(0)
    seeds = rng.integers(0, 256, (N_KEYS, 32), dtype=np.uint8)
    pks = eng.keygen_batch(seeds)
    assert eng.committee_register(pks).all()
    pre = np.frombuffer(rng.bytes(40 * N_MSGS), np.uint8).copy()
    off = (np.arange(N_MSGS + 1, dtype=np.uint64) * 40).astype(np.uint64)
    dig = eng.digest32_batch(pre, off)
    mi = rng.integers(0, N_MSGS, N_ITEMS).astype(np.uint32)
    kidx = rng.integers(0, N_KEYS, N_ITEMS).astype(np.uint32)
    modes = (np.arange(N_ITEMS) % 2).astype(np.uint8)
    sig = eng.sign_digests(seeds, pks, dig[mi], key_idx=kidx)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_pre, d_off, d_pk, d_mi, d_mode = t(pre), t(off.view(np.int64)), t(pks[kidx]), t(mi.view(np.int32)), t(modes)
    why = torch.empty(N_ITEMS, dtype=torch.uint8, device=dev)
    out = torch.empty(4, dtype=torch.int32, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    big = None
    for r in REJECTED:
        bad = np.sort(rng.choice(N_ITEMS, r, replace=False))
        s = sig.copy()
        s[bad, 0] ^= 1
        d_sig = t(s)
        ib = torch.zeros(N_ITEMS // 32, dtype=torch.int32, device=dev)
        eng.verify_groups_dev(d_pre, d_off, N_MSGS, d_sig, d_mi, ib, N_ITEMS, d_mode=d_mode, d_pk=d_pk)
        torch.cuda.synchronize()
        zeros = np.flatnonzero(np.unpackbits(ib.cpu().numpy().view(np.uint8), bitorder="little") == 0)
        assert (zeros == bad).all(), "the pass did not reject exactly the corrupted items"
        for cap in (0, 64):
            explain = lambda: eng.explain_groups_dev(d_pre, d_off, N_MSGS, d_sig, d_pk, d_mi, ib, N_ITEMS, why, out, d_mode=d_mode, max_explain=cap)
            explain()  # grows the scratch and checks the answer before anything is timed
            torch.cuda.synchronize()
            o = out.cpu().numpy().view(np.uint32)
            want = min(r, cap) if cap else r
            assert list(o) == [r, want, 0, 0xffffffff], o
            w = why.cpu().numpy()
            assert (w[bad[:want]] != 0x80).all() and (w == 0x80).sum() == N_ITEMS - want
            ms = []
            for _ in range(args.reps if r < 65536 or cap else max(3, args.reps // 2)):
                e0.record()
                explain()
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            emit(dict(workload="explain_after_pass", items=N_ITEMS, rejected=r, max_explain=cap, examined=want, **stats(ms)))
        if r == 65536:
            big = (d_sig, ib)
    # interference: 4,096-item passes on stream A, alone or beside a 65,536-item explanation on stream B
    d_sig, ib = big
    small = 4096
    sib = torch.zeros(small // 32, dtype=torch.int32, device=dev)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.passes)]
    arms = {"alone": [], "beside_explain_65536": []}

    def passes():
        with torch.cuda.stream(sa):
            for a, b in evs:
                a.record(sa)
                eng.verify_groups_dev(d_pre, d_off, N_MSGS, d_sig[:small], d_mi[:small], sib, small, d_mode=d_mode[:small], d_pk=d_pk[:small])
                b.record(sa)

    passes()
    torch.cuda.synchronize()
    expl_ms = []
    for rnd in range(2 * args.rounds):
        beside = rnd % 2 == 1
        torch.cuda.synchronize()
        if beside:
            with torch.cuda.stream(sb):
                x0, x1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                x0.record(sb)
                eng.explain_groups_dev(d_pre, d_off, N_MSGS, d_sig, d_pk, d_mi, ib, N_ITEMS, why, out, d_mode=d_mode)
                x1.record(sb)
        passes()
        torch.cuda.synchronize()
        arms["beside_explain_65536" if beside else "alone"] += [a.elapsed_time(b) for a, b in evs]
        if beside:
            expl_ms.append(x0.elapsed_time(x1))
    for arm, ms in arms.items():
        emit(dict(workload="groups_dev_4096_stream", arm=arm, rounds=args.rounds, passes_per_round=args.passes, **stats(ms)))
    emit(dict(workload="explain_65536_beside_passes", **stats(expl_ms)))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
