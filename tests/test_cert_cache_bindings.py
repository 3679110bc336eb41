"""The verify queue's certificate cache (hs_queue_cert_cache, hs_queue_cert_stats) in every binding against include/hs_crypto.h (CPU
only): the declarations, the ctypes table, the Python names, the Rust submodule's extern block and its use by verify_timeout_queued,
and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST_TO_C = dict(QUEUE_RUST_TO_C, **{"*mut u64": "uint64_t*"})


def test_header_declares_the_cert_cache():
    fns = header_functions()
    assert fns["hs_queue_cert_cache"] == ("int", ["hs_queue*", "size_t"])
    assert fns["hs_queue_cert_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_CERT_STATS 6\b", hdr)
    assert re.search(r"int hs_queue_cert_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_CERT_STATS\]\);", hdr)
    # the existing counters keep their layouts
    assert re.search(r"#define HS_QUEUE_STATS 6\b", hdr) and re.search(r"#define HS_QUEUE_DIGEST_STATS 4\b", hdr)


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import VerifyQueue
    assert _lib.SIGNATURES["hs_queue_cert_cache"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t])
    assert _lib.SIGNATURES["hs_queue_cert_stats"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    assert VerifyQueue.CERT_STATS == ("lookups", "hits", "joins", "records_answered", "inserted", "bytes_held")
    assert callable(VerifyQueue.cert_cache) and callable(VerifyQueue.cert_stats)


def test_rust_cert_cache_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_cert_cache.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_cert_cache.rs"\]\s*pub mod cert_cache;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_cert_cache", "hs_queue_cert_stats"}
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    assert "[0u64; 6]" in src and "== HS_OK" in src  # HS_QUEUE_CERT_STATS counters; a failed call is never read


def test_rust_timeout_goes_through_the_cached_queue():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_msgs_queue.rs")).read())
    assert re.search(r"pub async fn verify_timeout_queued\(", src)
    assert "cert_cache::enable(q)" in src
    # both entry points submit through the queue with the cache on; only verify_msgs_queued keeps the GROUP_MAX_SIGS cut-over
    assert src.count("cached_queue()?") == 1
    msgs = re.search(r"pub async fn verify_msgs_queued\(.*?\n\}", src, flags=re.S).group(0)
    assert "n > GROUP_MAX_SIGS" in msgs and "submit(" in msgs
    timeout = re.search(r"pub async fn verify_timeout_queued\(.*?\n\}", src, flags=re.S).group(0)
    assert "submit(" in timeout and "GROUP_MAX_SIGS" not in timeout


def test_cpp_cert_cache_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "cert.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  q.cert_cache(1 << 20);\n"
                   "  const std::array<uint64_t, HS_QUEUE_CERT_STATS> s = q.cert_stats();\n"
                   "  return s[0] == 0 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "cert")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
