"""hs_self_test: the on-device known-answer test of every device path at a context's own table geometry.

CPU: the vectors compiled into the library are exactly tests/golden/vectors.json.  GPU: the built-in set passes at several geometries,
with and without a committee; a wrong expectation is reported per path; the registered committee, the key cache and the verify queues
are left as they were, also while a queue is busy."""
import ctypes
import importlib.util
import os
import re
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_selftest_vectors.h")

HS_ERR_ARG, HS_ERR_SELFTEST = 2, 4


def _hs_defines():
    hdr = open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    d = {k: 1 << int(b) for k, b in re.findall(r"#define (HS_SELFTEST_\w+) \(1u << (\d+)\)", hdr)}
    d["HS_SELFTEST_VERIFY_PATHS"] = int(re.search(r"#define HS_SELFTEST_VERIFY_PATHS (0x[0-9a-f]+)u", hdr).group(1), 16)
    return d


def _generator():
    spec = importlib.util.spec_from_file_location("gen_selftest_vectors", os.path.join(ROOT, "tools", "gen_selftest_vectors.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_committed_header_is_the_generated_one(golden):
    assert open(HEADER).read() == _generator().render(golden), "rerun tools/gen_selftest_vectors.py"


def test_header_counts_match_the_golden_file(golden):
    text = open(HEADER).read()
    defs = dict((k, int(v)) for k, v in re.findall(r"#define (HS_ST_\w+) (\d+)", text))
    vs = golden["vectors"]
    assert defs["HS_ST_N_VECTORS"] == len(vs) and defs["HS_ST_N_DIGEST_KATS"] == len(golden["digest_kats"])
    assert defs["HS_ST_VEC_MSG_BYTES"] == sum(len(v["msg"]) // 2 for v in vs)
    assert defs["HS_ST_KAT_MSG_BYTES"] == sum(len(k["msg"]) // 2 for k in golden["digest_kats"])
    assert defs["HS_ST_N_SIGNATURES"] == 1 + len(golden["reference"]["qc_votes"]) and defs["HS_ST_N_SEEDS"] == len(golden["reference"]["seeds"])
    body = text.split("hs_st_vectors[HS_ST_N_VECTORS] = {")[1].split("};")[0]
    rows = re.findall(r'\{"([^"]+)", \{[^}]*\}, \{[^}]*\}, (\d+), (\d+), (\d)\},', body)
    assert [r[0] for r in rows] == [v["name"] for v in vs]
    assert [int(r[3]) for r in rows] == [int(v["strict"]) | 2 * int(v["batch_eq"]) for v in vs]
    assert [int(r[2]) for r in rows] == [len(v["msg"]) // 2 for v in vs]
    assert len({v["pk"] for v in vs}) == 39  # the distinct keys the scratch tables hold (hs_crypto.h sizes them)


def test_selftest_bits_are_distinct_and_verify_paths_cover_the_verify_kernels():
    d = _hs_defines()
    bits = [v for k, v in d.items() if k != "HS_SELFTEST_VERIFY_PATHS"]
    assert len(bits) == 15 and len(set(bits)) == 15 and all(b & (b - 1) == 0 for b in bits)
    verify = ("GENERIC", "VAR", "COMMITTEE", "LOOKUP", "MODES", "SMALL", "SMALL_CACHE", "BULK", "BULK_CACHE", "QUEUE_GENERIC")
    assert d["HS_SELFTEST_VERIFY_PATHS"] == sum(d["HS_SELFTEST_" + k] for k in verify)


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import build
    build.build_engine()


def _golden32(golden):
    vs = [v for v in golden["vectors"] if len(v["msg"]) == 64]
    recs = np.array([list(bytes.fromhex(v["sig"] + v["pk"] + v["msg"])) for v in vs], dtype=np.uint8)
    expect = np.array([int(v["strict"]) | 2 * int(v["batch_eq"]) for v in vs], dtype=np.uint8)
    return recs, expect


@pytest.mark.gpu
@pytest.mark.parametrize("base_window,key_window", [(24, 13), (24, 12), (20, 12), (16, 10), (26, 15)])
def test_builtin_set_passes_at_each_geometry(base_window, key_window):
    _gpu()
    from hotstuff_b200 import Engine
    e = Engine(0, base_window=base_window, key_window=key_window)
    try:
        launches = e.kernel_launches
        assert e.self_test() == 0, e.last_error
        assert e.kernel_launches > launches  # its launches count
        assert e.window_bits == (0, base_window) and e.cached_keys == 0
    finally:
        e.close()


@pytest.mark.gpu
def test_builtin_set_passes_with_and_without_a_committee_and_at_forced_windows(oracle):
    _gpu()
    from hotstuff_b200 import Engine
    e = Engine(0)
    try:
        assert e.self_test() == 0, e.last_error                         # fresh context: no committee, no key cache tables
        for kb in (8, 17):
            assert e.self_test(key_bits=kb) == 0, (kb, e.last_error)
        seeds = np.random.default_rng(11).integers(0, 256, (4096, 32), dtype=np.uint8)
        assert e.committee_register(oracle.keygen_batch(seeds)).all()
        assert e.self_test() == 0, e.last_error                         # at the committee's window
        for kb in (8, 17):
            assert e.self_test(key_bits=kb) == 0, (kb, e.last_error)
    finally:
        e.close()


@pytest.mark.gpu
def test_caller_vectors_report_a_flipped_expectation_on_every_verify_path(golden):
    _gpu()
    from hotstuff_b200 import Engine
    d = _hs_defines()
    recs, expect = _golden32(golden)
    e = Engine(0)
    try:
        assert e.self_test(recs=recs, expect=expect) == 0, e.last_error
        k = 6  # an even record: strict under the mixed mode bytes too, so every verify path sees the flip
        bad = expect.copy()
        bad[k] ^= 1
        failed = e.self_test(recs=recs, expect=bad)
        assert failed == d["HS_SELFTEST_VERIFY_PATHS"], hex(failed)
        assert "caller record %d" % k in e.last_error and "expected strict=%d" % (bad[k] & 1) in e.last_error, e.last_error
        assert e.self_test(recs=recs[:1], expect=expect[:1]) == 0, e.last_error   # one record, one key (every lookup a miss)
    finally:
        e.close()


@pytest.mark.gpu
def test_argument_errors(golden):
    _gpu()
    from hotstuff_b200 import Engine
    recs, expect = _golden32(golden)
    e = Engine(0)
    try:
        f = ctypes.c_uint32(0)
        p = recs.ctypes.data_as(ctypes.c_void_p)
        x = expect.ctypes.data_as(ctypes.c_void_p)
        st = e.lib.hs_self_test
        for kb in (-1, 7, 18, 24):
            assert st(e.h, kb, None, None, 0, ctypes.byref(f)) == HS_ERR_ARG
        assert st(e.h, 0, p, None, len(recs), ctypes.byref(f)) == HS_ERR_ARG         # records without expectations
        assert st(e.h, 0, None, x, 0, ctypes.byref(f)) == HS_ERR_ARG                 # expectations without records
        assert st(e.h, 0, None, None, 5, ctypes.byref(f)) == HS_ERR_ARG              # a size with the built-in set
        assert st(e.h, 0, p, x, 0, ctypes.byref(f)) == HS_ERR_ARG                    # no records
        big = np.zeros((4097, 128), np.uint8)
        assert st(e.h, 0, big.ctypes.data_as(ctypes.c_void_p), np.zeros(4097, np.uint8).ctypes.data_as(ctypes.c_void_p), 4097,
                  ctypes.byref(f)) == HS_ERR_ARG
        wrong = expect.copy()
        wrong[3] = 4
        assert st(e.h, 0, p, wrong.ctypes.data_as(ctypes.c_void_p), len(recs), ctypes.byref(f)) == HS_ERR_ARG
        assert st(e.h, 0, None, None, 0, None) == HS_ERR_ARG
        assert st(None, 0, None, None, 0, ctypes.byref(f)) == HS_ERR_ARG
        assert e.self_test() == 0, e.last_error
    finally:
        e.close()


@pytest.mark.gpu
def test_registered_committee_key_cache_and_queues_are_untouched(oracle):
    _gpu()
    from hotstuff_b200 import Engine
    from oracle_api import make_workload, to_rec128
    e = Engine(0)
    try:
        w = make_workload(oracle, 2048, n_keys=64, seed=21, corrupt_frac=0.1)
        recs = to_rec128(w)
        assert e.committee_register(w["pks"]).all()
        q = e.queue()
        q.sig_cache(1024)
        q.cert_cache(1 << 20)
        t = q.submit(recs[:8])
        assert (q.wait(t) == oracle.verify_rec128(recs[:8])).all()
        before = (e.verify_rec128(recs), e.verify_rec128(recs, mode=1), e.cached_keys, e.window_bits, q.stats(), q.digest_stats(),
                  q.sig_stats(), q.cert_stats(), q.generic_stats())
        assert (before[0] == oracle.verify_rec128(recs)).all()
        assert e.self_test() == 0 and e.self_test(key_bits=17) == 0, e.last_error
        after = (e.verify_rec128(recs), e.verify_rec128(recs, mode=1), e.cached_keys, e.window_bits, q.stats(), q.digest_stats(),
                 q.sig_stats(), q.cert_stats(), q.generic_stats())
        assert (before[0] == after[0]).all() and (before[1] == after[1]).all() and before[2:] == after[2:]
        q.close()
    finally:
        e.close()
    # the key cache: learned tables and their count are the same after the test
    e = Engine(0)
    try:
        w = make_workload(oracle, 512, n_keys=16, seed=22)
        recs = to_rec128(w)
        for _ in range(3):  # the key cache learns a pass's unknown keys at the start of a later call
            e.verify_rec128(recs)
        cached, wb = e.cached_keys, e.window_bits
        assert cached > 0
        assert e.self_test() == 0, e.last_error
        assert (e.cached_keys, e.window_bits) == (cached, wb)
        assert (e.verify_rec128(recs) == oracle.verify_rec128(recs)).all()
    finally:
        e.close()


@pytest.mark.gpu
def test_runs_while_eight_threads_push_votes_through_a_queue(oracle):
    _gpu()
    from hotstuff_b200 import Engine
    from oracle_api import make_workload, to_rec128
    e = Engine(0)
    try:
        w = make_workload(oracle, 1024, n_keys=32, seed=23, corrupt_frac=0.15)
        recs = to_rec128(w)
        want = oracle.verify_rec128(recs)
        assert e.committee_register(w["pks"]).all()
        q = e.queue()
        errors = []

        def voter(t):
            for i in range(t, len(recs), 8):
                if bool(q.wait(q.submit(recs[i:i + 1]))[0]) != bool(want[i]):
                    errors.append(i)

        th = [threading.Thread(target=voter, args=(t,)) for t in range(8)]
        for t in th:
            t.start()
        results = [e.self_test(), e.self_test(key_bits=8)]
        for t in th:
            t.join()
        assert results == [0, 0], e.last_error
        assert not errors, errors[:10]
        q.close()
    finally:
        e.close()
