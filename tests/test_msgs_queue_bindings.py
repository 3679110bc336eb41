"""The preimage path of the verify queue (hs_queue_submit_msgs, hs_queue_digest_stats) in every binding, against include/hs_crypto.h
(CPU only): the declarations, the Rust submodule's extern block and its callback, the ctypes table, the Python names, and the C++
wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MSGS_SIG = ("int", ["hs_queue*", "const uint8_t*", "const uint64_t*", "size_t", "const uint8_t*", "const uint8_t*", "const uint32_t*",
                    "const uint8_t*", "size_t", "hs_queue_cb*", "void*", "size_t*"])


def test_header_declares_submit_msgs_and_digest_stats():
    fns = header_functions()
    assert fns["hs_queue_submit_msgs"] == MSGS_SIG
    assert fns["hs_queue_digest_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_DIGEST_STATS 4\b", hdr) and re.search(r"#define HS_QUEUE_STATS 6\b", hdr)
    assert re.search(r"int hs_queue_digest_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_DIGEST_STATS\]\);", hdr)


def test_rust_msgs_queue_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_msgs_queue.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_msgs_queue.rs"\]\s*pub mod msgs_queue;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [QUEUE_RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert QUEUE_RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_submit_msgs"}
    called = set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, "")))
    assert called == seen
    # the node-wide queue, the header's callback type and the certificate cut-over are shared with the other queue modules
    assert re.search(r"use super::queue::\{[^}]*\bqueue\b[^}]*\bHsQueueCb\b[^}]*\};", src)
    assert re.search(r"use super::group_queue::GROUP_MAX_SIGS;", src)
    on_done = re.search(r"unsafe extern \"C\" fn on_done\((.*?)\)", src).group(1)
    assert [QUEUE_RUST_TO_C[p.split(":", 1)[1].strip()] for p in on_done.split(",")] == ["void*", "size_t", "int", "const uint32_t*"]
    # a failed submit is never an accept, an engine failure rejects every signature, and inconsistent arrays never reach the C ABI
    assert "if rc != HS_OK" in src and "status == HS_OK &&" in src
    assert re.search(r"n > GROUP_MAX_SIGS \|\| modes\.len\(\) != n \|\| sig\.len\(\) != 64 \* n \|\| pk\.len\(\) != 32 \* n", src)


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import VerifyQueue
    from hotstuff_b200 import wire
    ret, args = _lib.SIGNATURES["hs_queue_submit_msgs"]
    assert ret is ctypes.c_int and len(args) == len(MSGS_SIG[1])
    assert args[3] is ctypes.c_size_t and args[8] is ctypes.c_size_t and args[11] == ctypes.POINTER(ctypes.c_size_t)
    assert all(a is ctypes.c_void_p for k, a in enumerate(args[:11]) if k not in (3, 8))
    assert _lib.SIGNATURES["hs_queue_digest_stats"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    assert VerifyQueue.DIGEST_STATS == ("digest_launches", "preimages", "preimage_bytes", "msgs_requests")
    assert callable(VerifyQueue.submit_msgs) and callable(VerifyQueue.digest_stats) and callable(wire.submit_frame)


def test_cpp_submit_msgs_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "msgs.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  const uint8_t pre[16] = {};\n"
                   "  const uint64_t off[2] = {0, 16};\n"
                   "  uint8_t sig[2 * 64] = {}, pk[2 * 32] = {};\n"
                   "  const uint32_t idx[2] = {0, 0};\n"
                   "  const uint8_t modes[2] = {HS_MODE_STRICT, HS_MODE_BATCH_EQ};\n"
                   "  try {\n"
                   "    const bool ok = q.submit_msgs(pre, off, 1, sig, pk, idx, 2, modes).get().size() == 2;\n"
                   "    const std::array<uint64_t, HS_QUEUE_DIGEST_STATS> s = q.digest_stats();\n"
                   "    return ok && s[3] == 1 ? 0 : 1;\n"
                   "  } catch (const hs::QueueFull &) {\n"
                   "    return 2;\n"
                   "  }\n"
                   "}\n")
    out = str(tmp_path / "msgs")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
