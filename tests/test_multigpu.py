"""2-GPU check of the fused peer-store all-gather (include/hs_crypto.h hs_peer_*): each rank verifies its shard on its own
GPU and the finish kernel writes the bitmap words into BOTH ranks' buffers over NVLink; both ranks must end up with the
oracle's full bitmap.  Skipped on boxes with fewer than 2 GPUs (the driver's single-GPU run); the ncclAllGather baseline and
the sharding arithmetic are covered by tests/test_distributed.py on CPU (gloo)."""
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n, out_dir):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch
    import torch.distributed as dist
    from oracle_api import Oracle, make_workload, to_rec128
    from hotstuff_b200 import Engine
    from hotstuff_b200.sharding import PeerAllGather, all_gather_bitmap, shard_range
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    o = Oracle()
    w = make_workload(o, n, n_keys=11, seed=123, corrupt_frac=0.07, nthreads=4)
    recs = to_rec128(w)
    want = o.verify_rec128(recs, nthreads=4)
    e = Engine(rank, base_window=12)
    lo, hi, per = shard_range(n, rank, world)
    dev = torch.device("cuda", rank)
    d_recs = torch.from_numpy(recs[lo:hi]).to(dev)
    d_bm = torch.zeros((hi - lo + 31) // 32, dtype=torch.int32, device=dev)
    pag = PeerAllGather(e, n, rank, world)
    ok = True
    # Back-to-back epochs with DIFFERENT inputs per epoch and NO barrier / host synchronisation between them: every epoch's
    # gathered bitmap is snapshotted by a copy enqueued on the same stream right after the verify call (the documented
    # contract), while the other rank may already be one epoch ahead.  r1's single result buffer mixed epochs here; the
    # double buffer must not.  Rank 1 is slowed down on odd epochs and rank 0 on even ones to provoke both orders.
    n_epochs = 24
    variants = []
    for v in range(4):
        r2 = recs.copy()
        r2[v::7, 5] ^= np.uint8(1 << v)          # a different set of corrupted signatures per variant
        variants.append((torch.from_numpy(r2[lo:hi]).to(dev), o.verify_rec128(r2, nthreads=4)))
    snaps = []
    spin = torch.empty(1 << 22, dtype=torch.float32, device=dev)
    for ep in range(n_epochs):
        d_v, _ = variants[ep % 4]
        if (ep + rank) % 2 == 0:
            for _ in range(20):
                spin.normal_()                    # device-side delay on this rank only
        pag.arm()
        e.verify_rec128_dev(d_v, d_bm, hi - lo)
        snaps.append(pag.bitmap().clone())        # stream-ordered consumer of this epoch's bitmap
    torch.cuda.synchronize()
    for ep, snap in enumerate(snaps):
        got = np.unpackbits(snap.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
        ok = ok and bool((got == variants[ep % 4][1]).all())
    ok = ok and not e.lib.hs_peer_timed_out(e.h)
    dist.barrier()
    # an empty shard still takes part in the exchange (n == 0 on one rank)
    pag.arm()
    e.verify_rec128_dev(d_recs, d_bm, 0 if rank == 1 else hi - lo)
    torch.cuda.synchronize()
    ok = ok and not e.lib.hs_peer_timed_out(e.h)
    dist.barrier()
    # baseline path gives the same answer
    e.verify_rec128_dev(d_recs, d_bm, hi - lo)
    full = all_gather_bitmap(d_bm, n, world)
    got2 = np.unpackbits(full.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
    ok = ok and bool((got2 == want).all())
    np.save(os.path.join(out_dir, "ok_%d.npy" % rank), np.array([ok, (~want).sum() > 0]))
    dist.barrier()
    dist.destroy_process_group()
    e.close()


def test_peer_store_allgather_two_gpus(tmp_path):
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), 5000, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        res = np.load(os.path.join(str(tmp_path), "ok_%d.npy" % r))
        assert res[0] and res[1], "rank %d: gathered bitmap differs from the oracle" % r
