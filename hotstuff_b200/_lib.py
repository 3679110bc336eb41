"""ctypes binding of include/hs_crypto.h.  Loading fails loudly: there is no CPU fallback in the product."""
import ctypes
import os

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HS_CRYPTO_LIB") or os.path.join(PKG, "libhs_crypto.so")  # env override: kernel-variant experiments

c_void_p, c_size_t, c_u32, c_int, c_u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint64

# name -> (restype, argtypes); must list every symbol declared in include/hs_crypto.h
SIGNATURES = {
    "hs_ctx_create": (c_int, [ctypes.POINTER(c_void_p), c_int, c_u32]),
    "hs_ctx_destroy": (None, [c_void_p]),
    "hs_last_error": (ctypes.c_char_p, [c_void_p]),
    "hs_kernel_launches": (c_u64, [c_void_p]),
    "hs_cached_keys": (c_size_t, [c_void_p]),
    "hs_window_bits": (None, [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "hs_profile_enable": (c_int, [c_void_p, c_int]),
    "hs_profile_main_ms": (ctypes.c_double, [c_void_p]),
    "hs_host_alloc": (c_void_p, [c_size_t]),
    "hs_host_free": (None, [c_void_p]),
    "hs_verify_strict_batch": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_verify_rec128": (c_int, [c_void_p, c_void_p, c_size_t, c_u32, c_void_p]),
    "hs_verify_var": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_u32, c_void_p]),
    "hs_verify_batch_shared_msg": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, ctypes.POINTER(c_int), c_void_p]),
    "hs_verify_qcs": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_verify_tcs": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_verify_groups": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t,
                                 c_void_p, c_void_p]),
    "hs_verify_qc_votes_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_qc_and_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    "hs_verify_groups_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p,
                                     c_void_p]),
    "hs_explain_groups_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t,
                                      c_void_p, c_void_p, c_void_p]),
    "hs_ingest_consensus_frames": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_committee_register": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_committee_update": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]),
    "hs_committee_stage": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]),
    "hs_committee_commit": (c_int, [c_void_p]),
    "hs_committee_discard": (c_int, [c_void_p]),
    "hs_committee_stage_register": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_void_p]),
    "hs_set_table_budget": (c_int, [c_void_p, c_size_t]),
    "hs_verify_committee": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_u32, c_void_p]),
    "hs_digest32_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_verify_rec128_dev": (c_int, [c_void_p, c_void_p, c_size_t, c_u32, c_void_p, c_void_p]),
    "hs_verify_var_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_u32, c_void_p, c_void_p]),
    "hs_verify_committee_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_u32, c_void_p, c_void_p]),
    "hs_digest32_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_digest32_fixed_dev": (c_int, [c_void_p, c_void_p, c_size_t, c_size_t, c_void_p, c_void_p]),
    "hs_keygen_batch": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_sign_digests": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_keygen_batch_dev": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_sign_digests_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hs_set_deferred": (c_int, [c_void_p, c_int]),
    "hs_results_wait": (c_int, [c_void_p, c_void_p]),
    "hs_peer_setup": (c_int, [c_void_p, c_int, c_int, c_size_t, c_void_p]),
    "hs_peer_open": (c_int, [c_void_p, c_int, c_void_p]),
    "hs_peer_next": (c_int, [c_void_p, c_size_t, c_u32]),
    "hs_peer_bitmap": (c_void_p, [c_void_p]),
    "hs_peer_timed_out": (c_int, [c_void_p]),
    "hs_verify_msgs": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_u32, c_void_p]),
    "hs_verify_msgs_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_u32, c_void_p, c_void_p, c_void_p]),
    "hs_queue_create": (c_int, [c_void_p, c_size_t, ctypes.POINTER(c_void_p)]),
    "hs_queue_submit": (c_int, [c_void_p, c_void_p, c_size_t, c_u32, c_void_p, c_void_p, ctypes.POINTER(c_size_t)]),
    "hs_queue_submit_group": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, ctypes.POINTER(c_size_t)]),
    "hs_queue_poll": (c_int, [c_void_p, c_size_t, ctypes.POINTER(c_int), c_void_p]),
    "hs_queue_wait": (c_int, [c_void_p, c_size_t, c_void_p]),
    "hs_queue_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_submit_msgs": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p,
                                     ctypes.POINTER(c_size_t)]),
    "hs_queue_digest_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_cert_cache": (c_int, [c_void_p, c_size_t]),
    "hs_queue_cert_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_sig_cache": (c_int, [c_void_p, c_size_t]),
    "hs_queue_sig_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_sig_share": (c_int, [c_void_p, c_int]),
    "hs_queue_sig_share_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_sig_audit": (c_int, [c_void_p, c_size_t, c_size_t, ctypes.POINTER(c_u64)]),
    "hs_queue_sig_audit_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_generic": (c_int, [c_void_p, c_int]),
    "hs_queue_generic_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_batch": (c_int, [c_void_p, c_size_t, c_size_t]),
    "hs_queue_submit_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t,
                                      c_void_p, c_void_p, ctypes.POINTER(c_size_t)]),
    "hs_queue_batch_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_explain": (c_int, [c_void_p, c_size_t, c_size_t]),
    "hs_queue_submit_explain": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, ctypes.POINTER(c_size_t)]),
    "hs_queue_submit_explain_msgs": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p,
                                             ctypes.POINTER(c_size_t)]),
    "hs_queue_explain_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_queue_destroy": (None, [c_void_p]),
    "hs_self_test": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_size_t, ctypes.POINTER(c_u32)]),
    "hs_key_slots": (c_size_t, [c_void_p]),
    "hs_table_audit": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, ctypes.POINTER(c_u32)]),
    "hs_table_repair": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, ctypes.POINTER(c_u32), ctypes.POINTER(c_u32)]),
    "hs_table_mend": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, ctypes.POINTER(c_u32), ctypes.POINTER(c_u32)]),
    "hs_table_mend_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_scrub_mend": (c_int, [c_void_p, c_int]),
    "hs_scrub_start": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_u32, c_u32, c_u32, c_void_p, c_void_p]),
    "hs_scrub_set_map": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t]),
    "hs_scrub_stop": (c_int, [c_void_p]),
    "hs_scrub_stats": (c_int, [c_void_p, ctypes.POINTER(c_u64)]),
    "hs_scrub_sig_cache": (c_int, [c_void_p, c_void_p, c_u32]),
    "hs_explain_rec128": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_multi_create": (c_int, [ctypes.POINTER(c_void_p), c_void_p, c_size_t, c_u32]),
    "hs_multi_destroy": (None, [c_void_p]),
    "hs_multi_last_error": (ctypes.c_char_p, [c_void_p]),
    "hs_multi_members": (c_size_t, [c_void_p]),
    "hs_multi_member": (c_void_p, [c_void_p, c_size_t]),
    "hs_multi_committee_register": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "hs_multi_committee_update": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]),
    "hs_multi_verify_rec128": (c_int, [c_void_p, c_void_p, c_size_t, c_u32, c_void_p]),
    "hs_multi_verify_msgs": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_u32, c_void_p]),
    "hs_multi_verify_groups": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                       c_size_t, c_void_p, c_void_p]),
}

# hs_queue_cb: void (void *user, size_t ticket, int status, const uint32_t *bitmap)
QUEUE_CB = ctypes.CFUNCTYPE(None, c_void_p, c_size_t, c_int, ctypes.POINTER(c_u32))
# hs_scrub_cb: void (void *user, uint32_t found, uint32_t failed, size_t first_slot)
SCRUB_CB = ctypes.CFUNCTYPE(None, c_void_p, c_u32, c_u32, c_size_t)

_lib = None


def load():
    """Load libhs_crypto.so (built in-tree by hotstuff_b200.build).  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "hotstuff_b200: native CUDA library %s is missing — run `python -m hotstuff_b200.build` "
            "(there is no CPU fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
