"""The mend (hs_table_mend, hs_table_mend_stats, hs_scrub_mend) in every binding against include/hs_crypto.h (CPU only): the
declarations, the ctypes table, the Python names, the Rust submodule's extern block and its fall-back to the repair, and the C++
wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_scrub_bindings import RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEND_FNS = {"hs_table_mend", "hs_table_mend_stats", "hs_scrub_mend"}


def test_header_declares_the_mend():
    fns = header_functions()
    assert fns["hs_table_mend"] == ("int", ["hs_ctx*", "const uint8_t*", "const uint32_t*", "size_t", "uint8_t*", "uint32_t*", "uint32_t*"])
    assert fns["hs_table_mend_stats"] == ("int", ["hs_ctx*", "uint64_t*"])
    assert fns["hs_scrub_mend"] == ("int", ["hs_ctx*", "int"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_MEND_STATS 6\b", hdr)
    assert re.search(r"int hs_table_mend_stats\(hs_ctx \*ctx, uint64_t out\[HS_MEND_STATS\]\);", hdr)
    assert not any(n.startswith("hs_multi_") and "mend" in n for n in fns)  # a multi-device context is mended member by member


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import Engine
    c_void_p, c_size_t, c_u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32
    assert _lib.SIGNATURES["hs_table_mend"] == (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, ctypes.POINTER(c_u32),
                                                               ctypes.POINTER(c_u32)])
    assert _lib.SIGNATURES["hs_table_mend_stats"] == (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    assert _lib.SIGNATURES["hs_scrub_mend"] == (ctypes.c_int, [c_void_p, ctypes.c_int])
    assert Engine.MEND_STATS == ("calls", "windows_recomputed", "entries_rewritten", "windows_left", "slots_left", "cache_flushes")
    for name in ("table_mend", "mend_stats", "scrub_mend"):
        assert callable(getattr(Engine, name)), name


def test_rust_mend_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_mend.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_mend.rs"\]\s*pub mod mend;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == MEND_FNS
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen  # calls exactly what it declares
    assert "[0u64; 6]" in src and "== HS_OK" in src  # HS_MEND_STATS counters; a failed call is never read
    # what the mend leaves goes to the repair (audit_tables), which switches the GPU off if that fails
    body = re.search(r"pub fn mend_tables\(.*?\n\}", src, flags=re.S).group(0)
    assert re.search(r"if rc == HS_ERR_SELFTEST \{ return super::audit_tables\(expected\)", body)


def test_cpp_mend_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "mend.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  std::vector<std::array<uint8_t, 32>> keys(e.key_slots());\n"
                   "  uint32_t found = 0;\n"
                   "  std::vector<uint8_t> bits;\n"
                   "  uint32_t left = e.table_mend(&keys, nullptr, &found, &bits);\n"
                   "  e.scrub_mend(true);\n"
                   "  const std::array<uint64_t, HS_MEND_STATS> s = e.mend_stats();\n"
                   "  return (int)(left | found | (uint32_t)s[0]);\n"
                   "}\n")
    out = str(tmp_path / "mend")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
