"""Sharing of the verify queue's signature cache (hs_queue_sig_share, hs_queue_sig_share_stats) in every binding against
include/hs_crypto.h (CPU only): the declarations, the ctypes table, the Python names, the Rust submodule's extern block and where it
is turned on, and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST_TO_C = dict(QUEUE_RUST_TO_C, **{"*mut u64": "uint64_t*"})


def test_header_declares_the_sharing():
    fns = header_functions()
    assert fns["hs_queue_sig_share"] == ("int", ["hs_queue*", "int"])
    assert fns["hs_queue_sig_share_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_SIG_SHARE_STATS 5\b", hdr)
    assert re.search(r"int hs_queue_sig_share_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_SIG_SHARE_STATS\]\);", hdr)
    assert re.search(r"#define HS_QUEUE_SIG_STATS 5\b", hdr)  # the cache's own counters keep their layout


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import VerifyQueue
    assert _lib.SIGNATURES["hs_queue_sig_share"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int])
    assert _lib.SIGNATURES["hs_queue_sig_share_stats"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    assert VerifyQueue.SIG_SHARE_STATS == ("probed", "hits", "inserts", "evictions", "passes")
    assert callable(VerifyQueue.sig_share) and callable(VerifyQueue.sig_share_stats)


def test_rust_sig_share_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_sig_share.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_sig_share.rs"\]\s*pub mod sig_share;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_sig_share", "hs_queue_sig_share_stats"}
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    assert "[0u64; 5]" in src and "== HS_OK" in src  # HS_QUEUE_SIG_SHARE_STATS counters; a failed call is never read


def test_rust_shares_the_cache_right_after_turning_it_on():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_sig_cache.rs")).read())
    enable = re.search(r"pub\(crate\) fn enable\(.*?\n\}", src, flags=re.S).group(0)
    assert re.search(r"hs_queue_sig_cache\(q, SIG_CACHE_ENTRIES\) \}\s*== HS_OK\s*\{\s*super::sig_share::enable\(q\);", enable)


def test_cpp_sig_share_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "share.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  q.sig_cache(1 << 16);\n"
                   "  q.sig_share(true);\n"
                   "  const std::array<uint64_t, HS_QUEUE_SIG_SHARE_STATS> s = q.sig_share_stats();\n"
                   "  return s[4] == 0 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "share")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
