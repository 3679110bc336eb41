"""The staged committee change (hs_committee_stage, hs_committee_commit, hs_committee_discard) in every binding against
include/hs_crypto.h (CPU only): the declarations, the ctypes table, the Python names, the Rust shim, the C++ wrapper (which must compile
and link), and the one launch site of the table builder and the table prover.  A multi-device context stages member by member through
these single-context calls, so its C ABI keeps the hs_multi_ set it had; its bindings fan the three calls out over the members."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_launch_sites import LAUNCH, _code
from test_multi_bindings import MULTI_FUNCTIONS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_stage_commit_discard():
    fns = header_functions()
    assert fns["hs_committee_stage"] == fns["hs_committee_update"] == ("int", ["hs_ctx*", "const uint8_t*", "size_t", "const uint32_t*", "size_t",
                                                                               "uint32_t*"])
    assert fns["hs_committee_commit"] == fns["hs_committee_discard"] == ("int", ["hs_ctx*"])
    assert MULTI_FUNCTIONS == {f for f in fns if f.startswith("hs_multi_")}  # the multi-device ABI is unchanged


def test_ctypes_and_python_names():
    from hotstuff_b200 import Engine, MultiEngine, _lib
    P = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    assert _lib.SIGNATURES["hs_committee_stage"] == (ctypes.c_int, P)
    for name in ("hs_committee_commit", "hs_committee_discard"):
        assert _lib.SIGNATURES[name] == (ctypes.c_int, [ctypes.c_void_p]), name
    for name in ("committee_stage", "committee_commit", "committee_discard"):
        assert callable(getattr(Engine, name)), name
    for name in ("stage_committee", "commit_committee", "discard_committee"):
        assert callable(getattr(MultiEngine, name)), name
    assert not [n for n in _lib.SIGNATURES if n.startswith("hs_multi_") and n not in MULTI_FUNCTIONS]


def _fn_body(src, name):
    return re.search(r"pub fn %s\(.*?\n\}" % name, src, flags=re.S).group(0)


def test_rust_shim_stages_beside_keys_and_audits_after_the_commit():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    assert re.search(r"fn hs_committee_stage\(ctx: \*mut HsCtx, add_pks: \*const u8, n_add: usize, remove_idx: \*const u32, n_remove: usize, "
                     r"out_add_idx: \*mut u32\) -> c_int;", block)
    assert re.search(r"fn hs_committee_commit\(ctx: \*mut HsCtx\) -> c_int;", block)
    assert re.search(r"fn hs_committee_discard\(ctx: \*mut HsCtx\) -> c_int;", block)
    assert re.search(r"pub fn stage_committee\(add: &\[\[u8; 32\]\], remove_idx: &\[u32\]\) -> Result<Vec<u32>, GpuError>", src)
    for helper, fn in (("stage_on", "hs_committee_stage("), ("commit_on", "hs_committee_commit("), ("discard_on", "hs_committee_discard(")):
        body = re.search(r"\nfn %s\(.*?\n\}" % helper, src, flags=re.S).group(0)
        assert fn in body and "if rc != HS_OK { return Err(" in body, helper
    stage = _fn_body(src, "stage_committee")
    assert "KEYS" not in stage and "stage_on(c, add, remove_idx)?" in stage  # the map lists no staged index before the commit
    commit = _fn_body(src, "commit_committee")
    c, keys, audit = commit.index("commit_on(c)?"), commit.index("keys[i as usize] = Some(*k)"), commit.index("audit_tables(&keys)")
    assert c < keys < audit
    assert "STAGED.lock().unwrap() = None" in _fn_body(src, "update_committee")


def test_rust_multi_module_stages_member_by_member():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_multi.rs")).read())
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    assert set(re.findall(r"fn\s+(hs_\w+)", block)) == MULTI_FUNCTIONS
    stage = re.search(r"pub fn stage_committee\(.*?\n    \}", src, flags=re.S).group(0)
    assert "super::stage_on(" in stage and "std::thread::scope" in stage
    assert "super::discard_on(" in stage  # a failed or mismatched stage is discarded on every member
    assert "Some(x) if *x == v" in stage  # every member must return the same indices
    for fn, helper in (("commit_committee", "super::commit_on("), ("discard_committee", "super::discard_on(")):
        body = re.search(r"pub fn %s\(.*?\n    \}" % fn, src, flags=re.S).group(0)
        assert helper in body, fn


def test_cpp_wrappers_compile_and_link(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "stage.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  uint8_t pk[32] = {};\n"
                   "  uint32_t rem = 0;\n"
                   "  std::vector<uint32_t> idx = e.committee_stage(pk, 1, &rem, 1);\n"
                   "  e.committee_commit();\n"
                   "  e.committee_discard();\n"
                   "  hs::MultiEngine m({0, 0});\n"
                   "  idx = m.stage_committee(pk, 1, &rem, 1);\n"
                   "  m.commit_committee();\n"
                   "  m.discard_committee();\n"
                   "  return (int)idx.size();\n"
                   "}\n")
    out = str(tmp_path / "stage")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)


def test_table_builder_and_prover_have_one_launch_site():
    launches = [m.group(1) for m in LAUNCH.finditer(_code())]
    assert launches.count("k_build_comb") == 1 and launches.count("k_table_audit") == 1
    code = _code()
    for fn, kernel in (("launch_build", "k_build_comb"), ("launch_table_audit", "k_table_audit")):
        body = re.search(r"static int %s\(.*?\n\}" % fn, code, flags=re.S).group(0)
        assert re.search(r"\b%s\s*(?:<[^<>;]*>)?\s*<<<" % kernel, body), fn
