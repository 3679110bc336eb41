"""The engine-owned scrub (hs_scrub_start, hs_scrub_set_map, hs_scrub_stop, hs_scrub_stats) in every binding against
include/hs_crypto.h (CPU only): the declarations, the ctypes table and callback type, the Python names, the Rust submodule's extern
block and where the shim uses it, and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST_TO_C = dict(QUEUE_RUST_TO_C, **{"*mut u64": "uint64_t*", "Option<HsScrubCb>": "hs_scrub_cb*"})
SCRUB_FNS = {"hs_scrub_start", "hs_scrub_set_map", "hs_scrub_stop", "hs_scrub_stats"}


def test_header_declares_the_scrub():
    fns = header_functions()
    assert fns["hs_scrub_start"] == ("int", ["hs_ctx*", "const uint8_t*", "const uint32_t*", "size_t", "uint32_t", "uint32_t", "uint32_t",
                                             "hs_scrub_cb*", "void*"])
    assert fns["hs_scrub_set_map"] == ("int", ["hs_ctx*", "const uint8_t*", "const uint32_t*", "size_t"])
    assert fns["hs_scrub_stop"] == ("int", ["hs_ctx*"])
    assert fns["hs_scrub_stats"] == ("int", ["hs_ctx*", "uint64_t*"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_SCRUB_STATS 8\b", hdr)
    assert re.search(r"int hs_scrub_stats\(hs_ctx \*ctx, uint64_t out\[HS_SCRUB_STATS\]\);", hdr)
    assert re.search(r"typedef void\(hs_scrub_cb\)\(void \*user, uint32_t found, uint32_t failed, size_t first_slot\);", hdr)
    assert not any(n.startswith("hs_multi_scrub") for n in fns)  # a multi-device context is scrubbed member by member


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import Engine
    c_void_p, c_size_t, c_u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32
    assert _lib.SIGNATURES["hs_scrub_start"] == (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_u32, c_u32, c_u32, c_void_p, c_void_p])
    assert _lib.SIGNATURES["hs_scrub_set_map"] == (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_size_t])
    assert _lib.SIGNATURES["hs_scrub_stop"] == (ctypes.c_int, [c_void_p])
    assert _lib.SIGNATURES["hs_scrub_stats"] == (ctypes.c_int, [c_void_p, ctypes.POINTER(ctypes.c_uint64)])
    cb = _lib.SCRUB_CB
    assert cb._restype_ is None and list(cb._argtypes_) == [c_void_p, c_u32, c_u32, c_size_t]
    assert Engine.SCRUB_STATS == ("passes", "slots_audited", "base_entries_audited", "ticks", "findings", "slots_repaired",
                                  "failed_repairs", "ticks_paused")
    for name in ("scrub_start", "scrub_set_map", "scrub_stop", "scrub_stats"):
        assert callable(getattr(Engine, name)), name


def test_rust_scrub_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_scrub.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_scrub.rs"\]\s*pub mod scrub;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen <= SCRUB_FNS and {"hs_scrub_start", "hs_scrub_set_map"} <= seen
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen  # calls exactly what it declares
    cb = re.search(r"pub type HsScrubCb = unsafe extern \"C\" fn\((.*?)\);", src).group(1)
    assert [RUST_TO_C[p.split(":", 1)[1].strip()] for p in cb.split(",")] == ["void*", "uint32_t", "uint32_t", "size_t"]
    assert "[0u64; 8]" in src and "== HS_OK" in src  # HS_SCRUB_STATS counters; a failed call is never read
    # a failed repair switches the GPU off; a repaired finding does not
    on = re.search(r"unsafe extern \"C\" fn on_finding\(.*?\n\}", src, flags=re.S).group(0)
    assert re.search(r"if failed != 0 \{ DISABLED\.store\(true, Ordering::Release\); \}", on)


def test_rust_shim_gives_the_scrub_every_new_map():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    for fn in ("register_committee", "update_committee", "commit_committee"):
        body = re.search(r"pub fn %s\(.*?\n\}" % fn, src, flags=re.S).group(0)
        assert "scrub::set_map(c, &" in body, fn
        if "audit_tables(" in body:
            assert body.index("audit_tables(") < body.index("scrub::set_map(")  # the map is proved first


def test_cpp_scrub_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "scrub.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "static void on_finding(void *, uint32_t, uint32_t failed, size_t) { (void)failed; }\n"
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  std::vector<std::array<uint8_t, 32>> keys(e.key_slots());\n"
                   "  e.scrub_start(&keys, nullptr, 2000, 64, 1u << 18, on_finding, nullptr);\n"
                   "  e.scrub_set_map(&keys);\n"
                   "  const std::array<uint64_t, HS_SCRUB_STATS> s = e.scrub_stats();\n"
                   "  e.scrub_stop();\n"
                   "  return s[0] == 0 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "scrub")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
