"""The certificate path of the verify queue (hs_queue_submit_group) in every binding, against include/hs_crypto.h (CPU only): the
Rust submodule's extern block and its callback type, the ctypes table, and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GROUP_SIG = ("int", ["hs_queue*", "const hs_rec128*", "size_t", "const uint8_t*", "hs_queue_cb*", "void*", "size_t*"])


def test_header_declares_submit_group():
    assert header_functions()["hs_queue_submit_group"] == GROUP_SIG


def test_rust_group_queue_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_group_queue.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_group_queue.rs"\]\s*pub mod group_queue;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [QUEUE_RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert QUEUE_RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_submit_group"}
    called = set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, "")))
    assert called == seen
    # the node-wide queue and the callback type are the queue module's: one ring, one dispatcher, the header's callback
    assert re.search(r"use super::queue::\{[^}]*\bqueue\b[^}]*\bHsQueueCb\b[^}]*\};", src)
    qsrc = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_queue.rs")).read())
    assert re.search(r"pub\(crate\) fn queue\(\) -> Option<\*mut HsQueue>", qsrc)
    on_done = re.search(r"unsafe extern \"C\" fn on_done\((.*?)\)", src).group(1)
    assert [QUEUE_RUST_TO_C[p.split(":", 1)[1].strip()] for p in on_done.split(",")] == ["void*", "size_t", "int", "const uint32_t*"]
    # a failed submit is never an accept, an engine failure rejects every signature, and the cut-over bounds the request
    assert "if rc != HS_OK" in src and "status == HS_OK &&" in src
    assert re.search(r"pub const GROUP_MAX_SIGS: usize = [\d_]+;", src)
    assert re.search(r"recs\.len\(\) > GROUP_MAX_SIGS \|\| modes\.len\(\) != recs\.len\(\) \{ return None; \}", src)


def test_ctypes_submit_group():
    from hotstuff_b200 import _lib
    ret, args = _lib.SIGNATURES["hs_queue_submit_group"]
    assert ret is ctypes.c_int and len(args) == len(GROUP_SIG[1])
    assert args[2] is ctypes.c_size_t and all(a is ctypes.c_void_p for a in args[:2] + args[3:6])


def test_cpp_submit_group_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "group.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  hs_rec128 r[2] = {};\n"
                   "  const uint8_t modes[2] = {HS_MODE_STRICT, HS_MODE_BATCH_EQ};\n"
                   "  try {\n"
                   "    return q.submit_group(r, 2, modes).get().size() == 2 ? 0 : 1;\n"
                   "  } catch (const hs::QueueFull &) {\n"
                   "    return 2;\n"
                   "  }\n"
                   "}\n")
    out = str(tmp_path / "group")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
