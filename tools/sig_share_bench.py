#!/usr/bin/env python3
"""What sharing the verify queue's signature cache with the synchronous calls and the batch lane (hs_queue_sig_share) saves a view
change, and what it costs a normal round.

One context per committee size N (keys made and signatures signed on the GPU), f = (N - 1) / 3.  Each run starts from an empty table:
  - the N Timeouts' author records arrive through the queue (groups of 64 records, k_verify_small) or as one collected burst on the
    batch lane (hs_queue_submit_batch);
  - then the TC of N - f votes: queued as one request (hs_queue_submit_msgs) at and below 502 records, else hs_verify_tcs;
  - then the Block that carries that TC: author (strict) + QC of 2f + 1 votes (batch-eq) + the TC's votes, through hs_verify_groups.
A normal round: a Block with its QC only (author + 2f + 1 votes) through hs_verify_groups, at N = 1,000 and 10,000.
Runs alternate sharing off and on, --runs of each; p50 / p99 of the host clock around each call (every call ends in a synchronise),
and the hits each call scored.  Every verdict is checked against the first run's.  Every line carries the card's name, power limit
and SM clocks from a read-only nvidia-smi query made in the same run.

    python tools/sig_share_bench.py [--runs 20] [--out profiles/r02_sig_share.jsonl]
"""
import argparse
import hashlib
import json
import os
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from table_audit_bench import keys, smi  # noqa: E402

GROUP_MAX_SIGS = 502
TABLE = 1 << 16


def dig(pre):
    return np.frombuffer(hashlib.sha512(pre).digest()[:32], np.uint8)


def pct(xs, p):
    return float(np.percentile(np.asarray(xs) * 1e6, p))


class Round:
    """The messages of one view change at N validators, signed on the GPU."""

    def __init__(self, eng, seeds, pks, n, rng):
        f = (n - 1) // 3
        self.n, self.f, self.round = n, f, int(rng.integers(1 << 20, 1 << 40))
        hq = (self.round - 1 - rng.integers(0, 5, n)).astype(np.uint64)
        self.hq = hq
        self.tpre = [struct.pack("<QQ", self.round, int(h)) for h in hq]
        tdig = np.array([dig(p) for p in self.tpre])
        self.tsig = eng.sign_digests(seeds, pks, tdig, key_idx=np.arange(n, dtype=np.uint32))
        self.tpk = pks
        self.tc = np.arange(n - f)
        bpre, qpre = rng.bytes(200), rng.bytes(40)
        qk = rng.permutation(n)[:2 * f + 1].astype(np.uint32)
        a_sig = eng.sign_digests(seeds, pks, dig(bpre)[None], key_idx=np.array([0], np.uint32))
        q_sig = eng.sign_digests(seeds, pks, np.tile(dig(qpre), (len(qk), 1)), key_idx=qk)
        self.block = self.groups([bpre, qpre], np.concatenate([a_sig, q_sig]), np.concatenate([pks[:1], pks[qk]]),
                                 np.concatenate([[0], np.ones(len(qk))]), np.concatenate([[0], np.ones(len(qk))]), with_tc=True)
        self.block_qc = self.groups([bpre, qpre], np.concatenate([a_sig, q_sig]), np.concatenate([pks[:1], pks[qk]]),
                                    np.concatenate([[0], np.ones(len(qk))]), np.concatenate([[0], np.ones(len(qk))]), with_tc=False)

    def groups(self, pres, sig, pk, mi, modes, with_tc):
        if with_tc:
            pres = pres + [self.tpre[i] for i in self.tc]
            sig = np.concatenate([sig, self.tsig[self.tc]])
            pk = np.concatenate([pk, self.tpk[self.tc]])
            mi = np.concatenate([mi, 2 + np.arange(len(self.tc))])
            modes = np.concatenate([modes, np.zeros(len(self.tc))])
        off = np.zeros(len(pres) + 1, np.uint64)
        off[1:] = np.cumsum([len(p) for p in pres])
        return dict(pre=np.frombuffer(b"".join(pres), np.uint8), off=off, sig=sig, pk=pk, mi=mi.astype(np.uint32),
                    gi=np.zeros(len(mi), np.uint32), modes=modes.astype(np.uint8))

    def timeouts_req(self):
        n = self.n
        return dict(pre=np.frombuffer(b"".join(self.tpre), np.uint8), off=np.arange(n + 1, dtype=np.uint64) * 16, sig=self.tsig, pk=self.tpk,
                    mi=np.arange(n, dtype=np.uint32), gi=np.arange(n, dtype=np.uint32), modes=np.zeros(n, np.uint8))


def verify_groups(eng, b):
    return eng.verify_groups(b["pre"], b["off"], b["sig"], b["mi"], b["gi"], 1, mode=b["modes"], pk=b["pk"], want_items=True)[1]


def arrive(q, r, how):
    if how == "queue":
        for i in range(0, r.n, 64):
            recs = np.concatenate([r.tsig[i:i + 64], r.tpk[i:i + 64], np.array([dig(p) for p in r.tpre[i:i + 64]])], axis=1)
            q.wait(q.submit_group(recs, np.zeros(len(recs), np.uint8)))
    else:
        t = r.timeouts_req()
        while (tk := q.submit_batch(t["pre"], t["off"], t["sig"], t["pk"], t["mi"], t["gi"], r.n, modes=t["modes"])) is None:
            time.sleep(0.0005)
        q.wait(tk)


def tc_call(eng, q, r):
    idx = r.tc
    if len(idx) <= GROUP_MAX_SIGS:
        pre = np.frombuffer(b"".join(r.tpre[i] for i in idx), np.uint8)
        return q.wait(q.submit_msgs(pre, np.arange(len(idx) + 1, dtype=np.uint64) * 16, r.tsig[idx], r.tpk[idx], np.arange(len(idx), dtype=np.uint32),
                                    modes=np.zeros(len(idx), np.uint8)))
    return eng.verify_tcs(np.array([r.round], np.uint64), r.tsig[idx], r.hq[idx], tc_idx=np.zeros(len(idx), np.uint32), pk=r.tpk[idx], want_votes=True)[1]


def hits(q, before):
    s, c = q.sig_share_stats(), q.sig_stats()
    return s["hits"] - before[0]["hits"] + c["hits"] - before[1]["hits"]


def snap(q):
    return q.sig_share_stats(), q.sig_stats()


def run_size(Engine, n, runs, rng, card, out):
    eng = Engine(0)
    try:
        seeds, pks = keys(eng, n, 1000 + n)
        assert eng.committee_register(pks).all()
        r = Round(eng, seeds, pks, n, rng)
        q = eng.queue(ring_records=16384)
        q.batch(max(n, 1024), 4 << 20)
        ref = {}
        res = {}
        for it in range(2 * runs):
            share = it % 2 == 1
            for how in ("queue", "lane"):
                q.sig_cache(0)
                q.sig_cache(TABLE)
                if share:
                    q.sig_share(True)
                arrive(q, r, how)
                for name, call in (("tc", lambda: tc_call(eng, q, r)), ("block_tc", lambda: verify_groups(eng, r.block)),
                                   ("block_qc", lambda: verify_groups(eng, r.block_qc))):
                    if name == "block_qc" and (how == "lane" or n not in (1000, 10000)):
                        continue
                    b = snap(q)
                    t0 = time.perf_counter()
                    bits = call()
                    dt = time.perf_counter() - t0
                    key = (how if name != "block_qc" else "-", name)
                    assert bits.all() and (key not in ref or (ref[key] == bits).all())
                    ref[key] = bits
                    res.setdefault(key + (share,), []).append((dt, hits(q, b)))
        q.close()
        for (how, name, share), v in sorted(res.items(), key=str):
            ts = [x[0] for x in v[1:]] or [v[0][0]]  # the first run of each warms up
            line = dict(bench="sig_share", n=n, f=(n - 1) // 3, timeouts=how, call=name,
                        path=("queued" if name == "tc" and n - (n - 1) // 3 <= GROUP_MAX_SIGS else
                              "hs_verify_tcs" if name == "tc" else "hs_verify_groups"),
                        records=int(n - (n - 1) // 3 if name == "tc" else len(r.block["mi"]) if name == "block_tc" else len(r.block_qc["mi"])),
                        share=share, runs=len(ts), p50_us=round(pct(ts, 50), 1), p99_us=round(pct(ts, 99), 1),
                        hits=int(np.median([x[1] for x in v])), card=card)
            print(json.dumps(line), flush=True)
            out.write(json.dumps(line) + "\n")
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--sizes", default="100,1000,4000,10000")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r02_sig_share.jsonl"))
    a = ap.parse_args()
    from hotstuff_b200 import Engine
    card = smi()
    rng = np.random.default_rng(4242)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as out:
        for n in (int(x) for x in a.sizes.split(",")):
            run_size(Engine, n, a.runs, rng, card, out)


if __name__ == "__main__":
    main()
