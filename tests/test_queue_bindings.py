"""The verify queue's bindings against include/hs_crypto.h (CPU only): the Rust submodule's extern block (its own block: it passes a
callback and a user pointer), the callback type in Rust / ctypes / the header, and the C++ RAII wrapper + the burst driver, which
must compile and link against the library."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import RUST_TO_C, _strip_comments, header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUEUE_RUST_TO_C = dict(RUST_TO_C, **{
    "*mut HsQueue": "hs_queue*", "*mut *mut HsQueue": "hs_queue**", "Option<HsQueueCb>": "hs_queue_cb*", "*mut c_void": "void*",
    "*mut usize": "size_t*", "*const u32": "const uint32_t*",
})
QUEUE_FNS = {"hs_queue_create", "hs_queue_submit", "hs_queue_poll", "hs_queue_wait", "hs_queue_destroy"}


def _header():
    return _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())


def test_header_declares_the_queue():
    fns = header_functions()
    assert QUEUE_FNS <= set(fns)
    assert fns["hs_queue_submit"] == ("int", ["hs_queue*", "const hs_rec128*", "size_t", "uint32_t", "hs_queue_cb*", "void*", "size_t*"])
    assert fns["hs_queue_poll"] == ("int", ["hs_queue*", "size_t", "int*", "uint32_t*"])
    assert "hs_queue_cb" not in fns     # the callback typedef is not read as a function
    m = re.search(r"typedef void\s*\(hs_queue_cb\)\s*\(([^)]*)\)\s*;", _header())
    assert m and [re.sub(r"\w+$", "", p.strip()).strip().replace(" *", "*") for p in m.group(1).split(",")] == ["void*", "size_t", "int", "const uint32_t*"]


def test_rust_queue_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_queue.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_queue.rs"\]\s*pub mod queue;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        c_ret, c_types = fns[name]
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [QUEUE_RUST_TO_C[r] for r in r_types] == c_types, name
        assert QUEUE_RUST_TO_C[ret] == c_ret, name
        seen.add(name)
    assert seen == {"hs_queue_create", "hs_queue_submit"}
    called = set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, "")))
    assert called == seen
    # the callback alias has the header's parameter list
    cb = re.search(r"pub type HsQueueCb = unsafe extern \"C\" fn\((.*?)\);", src).group(1)
    assert [QUEUE_RUST_TO_C[p.split(":", 1)[1].strip()] for p in cb.split(",")] == ["void*", "size_t", "int", "const uint32_t*"]
    # a failed submit is never an accept, and an engine failure rejects every signature
    assert "if rc != HS_OK" in src and "status == HS_OK &&" in src


def test_ctypes_queue_callback_type():
    from hotstuff_b200 import _lib
    assert _lib.QUEUE_CB._restype_ is None
    assert _lib.QUEUE_CB._argtypes_ == (ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_uint32))
    assert QUEUE_FNS <= set(_lib.SIGNATURES)


def test_cpp_queue_wrapper_and_burst_driver_compile_and_link(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    out = str(tmp_path / "queue_burst")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-o", out, os.path.join(ROOT, "tests", "cpp", "queue_burst.cpp"), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
