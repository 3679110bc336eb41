"""The verify queue's counters (hs_queue_stats) in every binding against include/hs_crypto.h (CPU only): the declaration, the ctypes
table, the Python names and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_queue_stats():
    assert header_functions()["hs_queue_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_STATS 6\b", hdr)
    assert re.search(r"int hs_queue_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_STATS\]\);", hdr)


def test_ctypes_and_python_queue_stats():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import VerifyQueue
    ret, args = _lib.SIGNATURES["hs_queue_stats"]
    assert ret is ctypes.c_int and args == [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)]
    assert VerifyQueue.STATS == ("small_launches", "small_records", "bulk_launches", "bulk_records", "slow_requests", "slow_records")


def test_cpp_queue_stats_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "stats.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  const std::array<uint64_t, HS_QUEUE_STATS> s = q.stats();\n"
                   "  return s[2] == 0 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "stats")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
