"""The verify queue's batch lane (hs_queue_batch, hs_queue_submit_batch, hs_queue_batch_stats) in every binding against
include/hs_crypto.h (CPU only): the declarations, the Rust submodule's extern block, its callback and status handling, the ctypes
table, the Python names, and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH_SIG = ("int", ["hs_queue*", "const uint8_t*", "const uint64_t*", "size_t", "const uint8_t*", "const uint8_t*", "const uint32_t*",
                     "const uint32_t*", "const uint8_t*", "size_t", "size_t", "hs_queue_cb*", "void*", "size_t*"])


def test_header_declares_the_batch_lane():
    fns = header_functions()
    assert fns["hs_queue_batch"] == ("int", ["hs_queue*", "size_t", "size_t"])
    assert fns["hs_queue_submit_batch"] == BATCH_SIG
    assert fns["hs_queue_batch_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_BATCH_STATS 5\b", hdr)
    assert re.search(r"int hs_queue_batch_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_BATCH_STATS\]\);", hdr)
    # the existing counters keep their layouts
    assert re.search(r"#define HS_QUEUE_STATS 6\b", hdr) and re.search(r"#define HS_QUEUE_DIGEST_STATS 4\b", hdr)
    assert re.search(r"#define HS_QUEUE_CERT_STATS 6\b", hdr) and re.search(r"#define HS_QUEUE_SIG_STATS 5\b", hdr)
    assert re.search(r"#define HS_QUEUE_GENERIC_STATS 3\b", hdr)


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib, wire
    from hotstuff_b200.engine import VerifyQueue
    assert _lib.SIGNATURES["hs_queue_batch"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t])
    ret, args = _lib.SIGNATURES["hs_queue_submit_batch"]
    assert ret is ctypes.c_int and len(args) == len(BATCH_SIG[1])
    assert args[3] is ctypes.c_size_t and args[9] is ctypes.c_size_t and args[10] is ctypes.c_size_t
    assert args[13] == ctypes.POINTER(ctypes.c_size_t)
    assert all(a is ctypes.c_void_p for k, a in enumerate(args[:13]) if k not in (3, 9, 10))
    assert _lib.SIGNATURES["hs_queue_batch_stats"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    assert VerifyQueue.BATCH_STATS == ("passes", "items", "groups", "preimage_bytes", "outside_committee")
    assert callable(VerifyQueue.batch) and callable(VerifyQueue.submit_batch) and callable(VerifyQueue.batch_stats)
    assert callable(wire.submit_frames) and callable(wire.verify_frames_queued)


def test_rust_batch_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_batch_queue.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_batch_queue.rs"\]\s*pub mod batch_queue;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [QUEUE_RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert QUEUE_RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_batch", "hs_queue_submit_batch"}
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    assert re.search(r"use super::queue::\{[^}]*\bqueue\b[^}]*\bHsQueueCb\b[^}]*\};", src)
    on_done = re.search(r"unsafe extern \"C\" fn on_done\((.*?)\)", src).group(1)
    assert [QUEUE_RUST_TO_C[p.split(":", 1)[1].strip()] for p in on_done.split(",")] == ["void*", "size_t", "int", "const uint32_t*"]


def test_rust_status_handling_never_accepts_on_failure():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_batch_queue.rs")).read())
    # a failed submit returns None and frees the pending state; the callback reads verdicts only when the status is HS_OK, and an
    # engine failure is None (never a vector of accepts)
    assert re.search(r"if rc != HS_OK \{\s*drop\(unsafe \{ Box::from_raw\(user as \*mut Pending\) \}\);\s*return None;", src)
    on_done = re.search(r"unsafe extern \"C\" fn on_done\(.*?\n\}", src, flags=re.S).group(0)
    assert re.search(r"let out = if status == HS_OK \{.*?\} else \{\s*None\s*\};", on_done, flags=re.S)
    # the lane is turned on once, and only a successful hs_queue_batch counts as on
    enable = re.search(r"pub\(crate\) fn enable\(.*?\n\}", src, flags=re.S).group(0)
    assert "call_once" in enable and "hs_queue_batch(q, max_items, max_bytes) } == HS_OK" in enable
    fn = re.search(r"pub async fn verify_groups_queued\(.*?\n\}", src, flags=re.S).group(0)
    assert "if !enable(q, BATCH_MAX_ITEMS, BATCH_MAX_BYTES) { return None; }" in fn
    # inconsistent arrays never reach the C ABI
    assert re.search(r"n > BATCH_MAX_ITEMS \|\| group_idx\.len\(\) != n \|\| modes\.len\(\) != n \|\| sig\.len\(\) != 64 \* n \|\| pk\.len\(\) != 32 \* n", fn)
    assert "rx.await.ok().flatten()" in fn


def test_cpp_batch_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "batch.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  q.batch(1024, 1 << 20);\n"
                   "  const uint8_t pre[16] = {};\n"
                   "  const uint64_t off[2] = {0, 16};\n"
                   "  uint8_t sig[2 * 64] = {}, pk[2 * 32] = {};\n"
                   "  const uint32_t idx[2] = {0, 0}, grp[2] = {0, 1};\n"
                   "  const uint8_t modes[2] = {HS_MODE_STRICT, HS_MODE_BATCH_EQ};\n"
                   "  try {\n"
                   "    const hs::BatchVerdicts v = q.submit_batch(pre, off, 1, sig, pk, idx, grp, modes, 2, 2).get();\n"
                   "    const std::array<uint64_t, HS_QUEUE_BATCH_STATS> s = q.batch_stats();\n"
                   "    return v.groups.size() == 2 && v.items.size() == 2 && s[0] == 1 ? 0 : 1;\n"
                   "  } catch (const hs::QueueFull &) {\n"
                   "    return 2;\n"
                   "  }\n"
                   "}\n")
    out = str(tmp_path / "batch")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
