"""Multi-GPU sharding of independent signatures (SURVEY.md §8e): one process per GPU, contiguous index ranges whose
length is a multiple of 32 so bitmap words never straddle ranks, and ONE collective — an all-gather of the per-rank
accept bitmaps — so that every rank (every validator process) ends up with the full bitmap.  Backend-agnostic
(`nccl` on the GPUs, `gloo` in the CPU tests)."""
import numpy as np


def shard_range(n, rank, world):
    """Records [lo, hi) owned by `rank`; every shard but the last has ceil(n / world) rounded up to 32 records."""
    per = -(-n // world)
    per = (per + 31) // 32 * 32
    lo = min(n, rank * per)
    hi = min(n, lo + per)
    return lo, hi, per


def all_gather_bitmap(local_words, n, world, group=None):
    """local_words: int32/uint32 tensor with the shard's bitmap (ceil(shard/32) words).  Returns the full bitmap
    (ceil(n/32) words) on every rank.  Shards are padded to the common per-rank word count for the collective."""
    import torch
    import torch.distributed as dist
    per_words = shard_range(n, 0, world)[2] // 32
    buf = torch.zeros(per_words, dtype=local_words.dtype, device=local_words.device)
    buf[: local_words.numel()] = local_words
    if world == 1:
        return buf[: (n + 31) // 32]
    out = torch.empty(per_words * world, dtype=local_words.dtype, device=local_words.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    return out[: (n + 31) // 32]


def verify_sharded(verify_fn, n, rank, world, device=None, group=None):
    """verify_fn(lo, hi) -> uint32 numpy array / tensor of ceil((hi-lo)/32) words for records [lo, hi).
    Returns bool[n] (numpy) assembled from every rank's shard."""
    import torch
    lo, hi, _ = shard_range(n, rank, world)
    words = verify_fn(lo, hi) if hi > lo else np.zeros(0, dtype=np.uint32)
    if isinstance(words, np.ndarray):
        words = torch.from_numpy(words.view(np.int32).copy())
    if device is not None:
        words = words.to(device)
    full = all_gather_bitmap(words, n, world, group)
    return np.unpackbits(full.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)


def verify_groups_sharded(engine, d_pre, d_off, d_sig, d_msg_idx, d_group_idx, n_groups, d_group_bitmap, rank, world, d_mode=None,
                          d_pk=None, d_vidx=None, peer=None, group=None):
    """A mixed certificate burst (Blocks, Timeouts with their high_qcs, TCs: items of both verdict modes) sharded over ranks.  Every
    argument but the preimages (d_pre, d_off: given whole to every rank) is the FULL per-item device array; this rank verifies the items
    shard_range(n_items, rank, world) gives it through Engine.verify_groups_dev, whose finish kernel judges each item in its own mode, so
    the words it produces are final.  They reach every rank through `peer` (a PeerAllGather over n_items, armed here) or, without one,
    the ncclAllGather fallback.  The per-group AND then runs on every rank over the whole gathered item bitmap with the whole d_group_idx,
    so every rank ends with every group verdict in d_group_bitmap.  Returns the gathered item bitmap ((n_items + 31) // 32 words).
    Deferred mode works on both paths; the bitmaps are then complete after engine.results_wait().  With `peer`, the AND follows the finish
    kernel on the engine's tail stream.  On the fallback the collective runs on the caller's stream, which the tail stream does not wait
    for, so this call waits on the host for the gathered bitmap before it enqueues the AND, and makes the caller's stream wait for the
    AND: deferral hides nothing there."""
    import torch
    n = d_msg_idx.numel()
    lo, hi, per = shard_range(n, rank, world)
    shard = lambda t: None if t is None else t[lo:hi]
    d_local = torch.zeros(max(1, per // 32), dtype=torch.int32, device=d_msg_idx.device)
    if peer is not None:
        peer.arm()
    engine.verify_groups_dev(d_pre, d_off, d_off.numel() - 1, shard(d_sig), shard(d_msg_idx), d_local, hi - lo, d_mode=shard(d_mode), d_pk=shard(d_pk),
                             d_vidx=shard(d_vidx))
    if peer is not None:
        full = peer.bitmap()
    else:
        engine.results_wait()  # deferred mode: the words come from the engine's tail stream, the collective reads them on this one
        full = all_gather_bitmap(d_local[: (hi - lo + 31) // 32], n, world, group)
        if full.is_cuda:  # deferred mode runs the AND on the tail stream, which does not wait for the collective on this stream
            torch.cuda.current_stream(full.device).synchronize()
    engine.qc_and_dev(full, d_group_idx, n, n_groups, d_group_bitmap)
    if peer is None:
        engine.results_wait()  # `full` is torch memory: it may be reused in this stream's order only after the AND has read it
    return full


class PeerAllGather:
    """Fused all-gather of the accept bitmap: the verify finish kernel stores its words straight into every rank's result
    buffer over NVLink (include/hs_crypto.h, hs_peer_*).  `ncclAllGather` (all_gather_bitmap above) is the baseline it replaces."""

    def __init__(self, engine, n_total, rank, world):
        """Collective constructor (every rank calls it).  Raises RuntimeError ON EVERY RANK if any rank cannot set up or map
        the CUDA-IPC buffers, so callers can fall back to all_gather_bitmap() consistently."""
        import ctypes
        import torch
        import torch.distributed as dist
        self.e, self.rank, self.world, self.n = engine, rank, world, n_total
        self.per_words = shard_range(n_total, 0, world)[2] // 32
        self.total_words = self.per_words * world
        torch.cuda.synchronize()
        dist.barrier()                      # a previous PeerAllGather on this engine is released by hs_peer_setup: nobody may still use it
        h = (ctypes.c_uint8 * 64)()
        ok = engine.lib.hs_peer_setup(engine.h, rank, world, self.total_words, h) == 0
        handles = [None] * world
        dist.all_gather_object(handles, bytes(h) if ok else None)
        if ok and all(x is not None for x in handles):
            for p, hp in enumerate(handles):
                if p != rank:
                    buf = (ctypes.c_uint8 * 64).from_buffer_copy(hp)
                    ok = ok and engine.lib.hs_peer_open(engine.h, p, buf) == 0
        else:
            ok = False
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=torch.device("cuda", engine.device))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            raise RuntimeError("peer buffers could not be set up on every rank: " + engine.lib.hs_last_error(engine.h).decode())
        self.epoch = 0
        ptr = engine.lib.hs_peer_bitmap(engine.h)   # epoch 0 -> first half of the double buffer
        # zero-copy torch view of this rank's result buffer: [2][total_words], indexed by epoch parity
        class _Arr:
            __cuda_array_interface__ = {"shape": (2, self.total_words), "typestr": "<i4", "data": (int(ptr), False), "version": 3}
        self._both = torch.as_tensor(_Arr(), device=torch.device("cuda", engine.device))

    def arm(self):
        """Call right before the engine's `_dev` verify of this rank's shard."""
        self.epoch += 1
        self.e._check(self.e.lib.hs_peer_next(self.e.h, self.rank * self.per_words, self.epoch), "hs_peer_next")

    @property
    def full(self):
        """All total_words of the most recently armed epoch (this rank's copy of every rank's verdicts)."""
        return self._both[self.epoch & 1]

    def bitmap(self):
        """The (n+31)//32 meaningful words.  Consume it (same stream) before arming the next epoch + 1 verify: the buffer is
        double-buffered by epoch parity, so no cross-rank barrier is needed between epochs."""
        return self.full[: (self.n + 31) // 32]
