"""The multi-device context's bindings (hs_multi_*, include/hs_crypto.h) against the header: the Rust submodule (source only: no Rust
toolchain here) by name, arity and parameter types, the Python wrapper, and the C++ wrapper by compiling and linking it.  CPU only."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import RUST_TO_C, _strip_comments, header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MULTI_RUST_TO_C = dict(RUST_TO_C, **{
    "*mut HsMulti": "hs_multi*", "*const HsMulti": "const hs_multi*", "*mut *mut HsMulti": "hs_multi**", "*const c_int": "const int*",
    "*const c_char": "const char*", "": "void",
})
MULTI_FUNCTIONS = {"hs_multi_create", "hs_multi_destroy", "hs_multi_last_error", "hs_multi_members", "hs_multi_member",
                   "hs_multi_committee_register", "hs_multi_committee_update", "hs_multi_verify_rec128", "hs_multi_verify_msgs",
                   "hs_multi_verify_groups"}


def test_header_declares_the_multi_context():
    fns = header_functions()
    assert MULTI_FUNCTIONS == {f for f in fns if f.startswith("hs_multi_")}
    assert fns["hs_multi_create"] == ("int", ["hs_multi**", "const int*", "size_t", "uint32_t"])
    assert fns["hs_multi_member"] == ("hs_ctx*", ["hs_multi*", "size_t"])
    # the sharded calls take exactly the single-context calls' arguments after the handle
    for name in ("verify_rec128", "verify_msgs", "verify_groups"):
        assert fns["hs_multi_" + name][1][1:] == fns["hs_" + name][1][1:], name
        assert fns["hs_multi_" + name][0] == fns["hs_" + name][0] == "int"
    for name in ("committee_register", "committee_update"):
        assert fns["hs_multi_" + name][1][1:] == fns["hs_" + name][1][1:], name
    hdr = open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    assert re.search(r"#define HS_MULTI_MIN_SHARD 4096\b", hdr)


def test_rust_multi_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_multi.rs")).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_multi.rs"\]\s*pub mod multi;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        assert name in fns, "%s is not declared in include/hs_crypto.h" % name
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert len(r_types) == len(fns[name][1]), "%s: %d parameters in the module, %d in the header" % (name, len(r_types), len(fns[name][1]))
        for k, (r, c) in enumerate(zip(r_types, fns[name][1])):
            assert MULTI_RUST_TO_C[r] == c, "%s parameter %d: module %r vs header %r" % (name, k, r, c)
        assert MULTI_RUST_TO_C[ret] == fns[name][0], "%s: return type" % name
        seen.add(name)
    assert seen == MULTI_FUNCTIONS
    # every declared function is called, and the main shim's extern block is unchanged: it declares none of them
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    shim_block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', _strip_comments(shim), flags=re.S).group(1)
    assert "hs_multi" not in shim_block


def test_rust_multi_module_never_accepts_on_failure():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_multi.rs")).read())
    for fn in ("verify_rec128", "verify_msgs"):
        body = re.search(r"pub fn %s\(.*?\n    \}" % fn, src, flags=re.S).group(0)
        assert re.search(r"if rc == HS_OK \{ bits\(&bm, [\w.()]+\) \} else \{ vec!\[false; [\w.()]+\] \}", body), fn
    body = re.search(r"pub fn verify_ingested\(.*?\n    \}", src, flags=re.S).group(0)
    assert "rc == HS_OK &&" in body
    for fn in ("register_committee", "update_committee"):
        body = re.search(r"pub fn %s\(.*?\n    \}" % fn, src, flags=re.S).group(0)
        assert "if rc != HS_OK { return Err(self.err()); }" in body, fn


def test_python_multi_engine_binds_every_function():
    from hotstuff_b200 import MultiEngine, _lib
    for name in MULTI_FUNCTIONS:
        assert name in _lib.SIGNATURES, name
    assert _lib.SIGNATURES["hs_multi_member"] == (ctypes.c_void_p, [ctypes.c_void_p, ctypes.c_size_t])
    assert MultiEngine.MIN_SHARD == 4096
    for m in ("register_committee", "update_committee", "verify_rec128", "verify_msgs", "verify_groups", "member", "close"):
        assert callable(getattr(MultiEngine, m)), m


def test_cpp_multi_engine_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "multi.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::MultiEngine m({0, 0}, 16 | (12 << 8));\n"
                   "  hs::VerifyQueue q(m.member(0));\n"
                   "  uint8_t pk[32] = {};\n"
                   "  const std::vector<uint32_t> valid = m.register_committee(pk, 1);\n"
                   "  hs_rec128 r{};\n"
                   "  const std::vector<uint32_t> bm = m.verify_rec128(&r, 1);\n"
                   "  return valid.size() == 1 && bm.size() == 1 && m.size() == 2 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "multi")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
