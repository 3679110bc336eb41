"""Wire-format ingest (SURVEY §8f.3): bincode `ConsensusMessage` frames -> the flat arrays `Engine.verify_groups` consumes, through
the C ABI's hs_ingest_consensus_frames (hotstuff_b200/csrc/hs_ingest.cpp).  Replaces, for the crypto path, the reference's
bincode::deserialize + per-signature walk (consensus/src/consensus.rs:33-39,138; crypto/src/lib.rs:94-112,178-182)."""
import ctypes
import threading

import numpy as np

from . import _lib

KIND_PROPOSE, KIND_VOTE, KIND_TIMEOUT, KIND_TC, KIND_SYNC_REQUEST, KIND_MALFORMED = 0, 1, 2, 3, 4, 255
NO_ITEM = 0xFFFFFFFF

FRAME_INFO = np.dtype([("kind", np.uint8), ("has_tc", np.uint8), ("qc_is_genesis", np.uint8), ("pad", np.uint8), ("author_item", np.uint32),
                       ("qc_lo", np.uint32), ("qc_hi", np.uint32), ("tc_lo", np.uint32), ("tc_hi", np.uint32),
                       ("round", np.uint64), ("qc_round", np.uint64), ("tc_round", np.uint64)])
assert FRAME_INFO.itemsize == 48


class _IngestOut(ctypes.Structure):
    _fields_ = [("cap_items", ctypes.c_size_t), ("cap_msgs", ctypes.c_size_t), ("cap_pre_bytes", ctypes.c_size_t),
                ("sig", ctypes.c_void_p), ("pk", ctypes.c_void_p), ("msg_idx", ctypes.c_void_p), ("group_idx", ctypes.c_void_p),
                ("mode", ctypes.c_void_p), ("preimages", ctypes.c_void_p), ("pre_off", ctypes.c_void_p),
                ("n_items", ctypes.c_size_t), ("n_msgs", ctypes.c_size_t), ("pre_bytes", ctypes.c_size_t)]


def ingest_frames(frames):
    """frames: list of bytes (one bincode ConsensusMessage each).  Returns dict(info, sig, pk, msg_idx, group_idx, mode, preimages,
    pre_off): frame i is group i; info[i] (FRAME_INFO) says which items are its author signature / QC votes / TC votes."""
    lib = _lib.load()
    n = len(frames)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(f) for f in frames])
    blob = np.frombuffer(b"".join(frames), dtype=np.uint8) if n and off[-1] else np.zeros(1, np.uint8)
    info = np.zeros(max(1, n), dtype=FRAME_INFO)
    total = int(off[-1])
    # every item costs >= 116 frame bytes, every preimage is copied from frame bytes: generous first guess, exact retry on NOMEM
    cap_items, cap_msgs, cap_pre = total // 116 + n + 1, total // 60 + n + 1, total + 64 * n + 64
    for _ in range(2):
        bufs = dict(sig=np.zeros((cap_items, 64), np.uint8), pk=np.zeros((cap_items, 32), np.uint8), msg_idx=np.zeros(cap_items, np.uint32),
                    group_idx=np.zeros(cap_items, np.uint32), mode=np.zeros(cap_items, np.uint8), preimages=np.zeros(cap_pre, np.uint8),
                    pre_off=np.zeros(cap_msgs + 1, np.uint64))
        o = _IngestOut(cap_items, cap_msgs, cap_pre, *(bufs[k].ctypes.data for k in ("sig", "pk", "msg_idx", "group_idx", "mode", "preimages", "pre_off")), 0, 0, 0)
        rc = lib.hs_ingest_consensus_frames(blob.ctypes.data, off.ctypes.data, n, info.ctypes.data, ctypes.byref(o))
        if rc == 0:
            ni, nm = o.n_items, o.n_msgs
            return dict(info=info[:n], sig=bufs["sig"][:ni], pk=bufs["pk"][:ni], msg_idx=bufs["msg_idx"][:ni], group_idx=bufs["group_idx"][:ni],
                        mode=bufs["mode"][:ni], preimages=bufs["preimages"][:o.pre_bytes], pre_off=bufs["pre_off"][:nm + 1], n_frames=n)
        if rc != 3:
            raise ValueError("hs_ingest_consensus_frames: status %d" % rc)
        cap_items, cap_msgs, cap_pre = o.n_items + 1, o.n_msgs + 1, o.pre_bytes + 1
    raise RuntimeError("ingest capacity retry failed")


def submit_frame(queue, frame, callback=None):
    """Ingests ONE frame and submits every signature in it to a VerifyQueue as one request (VerifyQueue.submit_msgs, preimages
    hashed on the GPU).  Returns None when the frame carries no signature (a SyncRequest, a malformed frame: nothing is submitted),
    else (info, ticket): info is the frame's FRAME_INFO, ticket None when the queue has no room now.  The verdicts are per item in
    ingest order; the frame's certificates hold iff they all do.  The stake / duplicate pre-checks stay with the caller."""
    g = ingest_frames([frame])
    if len(g["sig"]) == 0:
        return None
    return g["info"][0], queue.submit_msgs(g["preimages"], g["pre_off"], g["sig"], g["pk"], g["msg_idx"], modes=g["mode"], callback=callback)


def submit_frames(queue, frames, callback=None):
    """Ingests many frames and submits every signature in them to a VerifyQueue's batch lane as ONE request
    (VerifyQueue.submit_batch, group = frame).  Returns (ingest, ticket): ingest is what ingest_frames returns, ticket None when the
    frames carry no signature (nothing is submitted) or the lane has no room now.  The verdicts are (frame bools, item bools in
    ingest order); a frame without items is True.  The stake / duplicate pre-checks stay with the caller (verify_frames_queued)."""
    g = ingest_frames(frames)
    if len(g["sig"]) == 0:
        return g, None
    return g, queue.submit_batch(g["preimages"], g["pre_off"], g["sig"], g["pk"], g["msg_idx"], g["group_idx"], g["n_frames"], modes=g["mode"],
                                 callback=callback)


def verify_frames(frames, committee, engine):
    """Ingest + the reference's pre-checks + ONE engine pass.  Returns a list: None (valid), "Malformed", or the ConsensusError name
    the reference would raise first (same order as messages.verify_blocks).  SyncRequest frames are None (nothing to verify)."""
    def run(g, keep, n):
        return engine.verify_groups(g["preimages"], g["pre_off"], g["sig"][keep], g["msg_idx"][keep], g["group_idx"][keep], n, mode=g["mode"][keep],
                                    pk=g["pk"][keep], want_items=True)[1]
    return _verify_frames(frames, committee, run)


def verify_frames_queued(frames, committee, queue):
    """verify_frames with the pass on a VerifyQueue's batch lane (VerifyQueue.submit_batch): the same pre-checks, error names and error
    order.  Waits for the lane when its arena has no room."""
    def run(g, keep, n):
        while (t := queue.submit_batch(g["preimages"], g["pre_off"], g["sig"][keep], g["pk"][keep], g["msg_idx"][keep], g["group_idx"][keep], n,
                                       modes=g["mode"][keep])) is None:
            threading.Event().wait(0.0005)  # no room now: back-pressure
        return queue.wait(t)[1]
    return _verify_frames(frames, committee, run)


def _verify_frames(frames, committee, run):
    """The pre-checks and verdict order of verify_frames; run(ingest, kept items mask, n_frames) -> item bools of the kept items."""
    g = ingest_frames(frames)
    info, pk = g["info"], g["pk"]
    n = g["n_frames"]
    out = [None] * n
    skip = np.zeros(len(g["sig"]), dtype=bool)       # items whose certificate failed a pre-check are not judged
    qc_err, tc_err = [None] * n, [None] * n

    def quorum(lo, hi, err):
        weight, used = 0, set()
        for i in range(lo, hi):
            k = pk[i].tobytes()
            if k in used:
                return "AuthorityReuse"
            st = committee.stakes.get(k, 0)
            if st <= 0:
                return "UnknownAuthority"
            used.add(k)
            weight += st
        return None if weight >= committee.quorum_threshold() else err

    for j in range(n):
        f = info[j]
        if f["kind"] == KIND_MALFORMED:
            out[j] = "Malformed"
            continue
        if f["author_item"] != NO_ITEM and committee.stakes.get(pk[f["author_item"]].tobytes(), 0) <= 0:
            out[j] = "UnknownAuthority"
            skip[f["qc_lo"]:f["qc_hi"]] = True
            skip[f["tc_lo"]:f["tc_hi"]] = True
            skip[f["author_item"]] = True
            continue
        if f["kind"] in (KIND_PROPOSE, KIND_TIMEOUT) and not f["qc_is_genesis"]:
            qc_err[j] = quorum(f["qc_lo"], f["qc_hi"], "QCRequiresQuorum")
            if qc_err[j]:
                skip[f["qc_lo"]:f["qc_hi"]] = True
                skip[f["tc_lo"]:f["tc_hi"]] = True
        if f["has_tc"] and not qc_err[j]:
            tc_err[j] = quorum(f["tc_lo"], f["tc_hi"], "TCRequiresQuorum")
            if tc_err[j]:
                skip[f["tc_lo"]:f["tc_hi"]] = True
    keep = ~skip
    items = np.zeros(len(skip), dtype=bool)
    if keep.any():
        items[keep] = run(g, keep, n)
    for j in range(n):
        f = info[j]
        if out[j] is not None or f["kind"] == KIND_SYNC_REQUEST:
            continue
        if f["author_item"] != NO_ITEM and not items[f["author_item"]]:
            out[j] = "InvalidSignature"
        elif qc_err[j]:
            out[j] = qc_err[j]
        elif not items[f["qc_lo"]:f["qc_hi"]].all():
            out[j] = "InvalidSignature"
        elif tc_err[j]:
            out[j] = tc_err[j]
        elif not items[f["tc_lo"]:f["tc_hi"]].all():
            out[j] = "InvalidSignature"
    return out
