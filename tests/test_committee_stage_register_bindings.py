"""The staged registration (hs_committee_stage_register) in every binding against include/hs_crypto.h (CPU only): the declaration, the
ctypes table, the Python names, the Rust submodule and multi::Multi, the C++ wrapper (which must compile and link), and the one launch
site of the table builder and of both audit kernels, which prove the staged store as they prove the live one.  The multi-device C ABI
keeps the hs_multi_ set it had: a multi-device context stages a registration member by member."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_launch_sites import LAUNCH, _code
from test_multi_bindings import MULTI_FUNCTIONS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_stage_register():
    fns = header_functions()
    assert fns["hs_committee_stage_register"] == ("int", ["hs_ctx*", "const uint8_t*", "size_t", "int", "uint32_t*", "int*"])
    assert MULTI_FUNCTIONS == {f for f in fns if f.startswith("hs_multi_")}
    h = open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    doc = h[h.index("/* Staged registration"):h.index("int hs_committee_stage_register(")]
    for phrase in ("- Rule: hs_committee_stage_register(P, w) followed by hs_committee_commit", "HS_ERR_NOMEM", "HS_ERR_SELFTEST", "HS_ERR_ARG",
                   "_dev` verify pass"):
        assert phrase in doc, phrase


def test_ctypes_and_python_names():
    from hotstuff_b200 import Engine, MultiEngine, _lib
    assert _lib.SIGNATURES["hs_committee_stage_register"] == (
        ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p])
    assert callable(Engine.committee_stage_register) and callable(MultiEngine.stage_register_committee)
    assert not [n for n in _lib.SIGNATURES if n.startswith("hs_multi_") and n not in MULTI_FUNCTIONS]


def test_rust_submodule_and_multi():
    shim = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    assert '#[path = "crypto_gpu_stage_register.rs"]' in shim and "pub mod stage_register;" in shim
    assert "pub use stage_register::{commit_registration, discard_registration, stage_register_committee};" in shim
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_stage_register.rs")).read())
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    assert set(re.findall(r"fn\s+(hs_\w+)", block)) == {"hs_committee_stage_register"}
    assert re.search(r"fn hs_committee_stage_register\(ctx: \*mut HsCtx, pks: \*const u8, n: usize, key_bits: c_int, out_valid_bitmap: \*mut u32,\s*"
                     r"out_key_bits: \*mut c_int\) -> c_int;", block)
    commit = re.search(r"pub fn commit_registration\(.*?\n\}", src, flags=re.S).group(0)
    c, keys, scrub = commit.index("commit_on(c)?"), commit.index("*keys = staged"), commit.index("scrub::set_map(c, &keys)")
    assert c < keys < scrub  # the map is replaced only once the engine switched, then handed to the scrub
    multi = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_multi.rs")).read())
    stage = re.search(r"pub fn stage_register_committee\(.*?\n    \}", multi, flags=re.S).group(0)
    assert "super::stage_register::stage_register_on(" in stage and "std::thread::scope" in stage
    assert "super::discard_on(" in stage and "Some(x) if *x == v" in stage


def test_cpp_wrappers_compile_and_link(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "stage_register.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  uint8_t pk[32] = {};\n"
                   "  std::pair<std::vector<uint32_t>, int> r = e.committee_stage_register(pk, 1, 12);\n"
                   "  e.committee_commit();\n"
                   "  hs::MultiEngine m({0, 0});\n"
                   "  r = m.stage_register_committee(pk, 1);\n"
                   "  m.commit_committee();\n"
                   "  return r.second;\n"
                   "}\n")
    out = str(tmp_path / "stage_register")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)


def test_builder_and_audit_kernels_keep_one_launch_site():
    launches = [m.group(1) for m in LAUNCH.finditer(_code())]
    for k in ("k_build_comb", "k_table_audit", "k_slot_audit"):
        assert launches.count(k) == 1, k
    body = re.search(r"static int launch_slot_audit\(.*?\n\}", _code(), flags=re.S).group(0)
    assert re.search(r"\bk_slot_audit\s*<<<", body)
    code = _code()
    stage = re.search(r"int hs_committee_stage_register\(.*?\n\}\n", code, flags=re.S).group(0)
    for call in ("launch_build(", "launch_slot_audit(", "launch_table_audit(", "make_key_store("):
        assert call in stage, call


def test_rust_shim_keeps_one_record_of_the_engine_stage():
    """The engine has one stage slot of either kind: the shim mirrors it in one record, clears it on a registration or update, and each
    commit or discard checks the kind before it calls the engine and forgets the stage only once the engine's commit succeeded."""
    shim = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    sub = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_stage_register.rs")).read())
    assert re.search(r"enum Staged \{\s*Change \{[^}]*\},\s*Registration\(Vec<\[u8; 32\]>\),\s*\}", shim)
    assert len(re.findall(r"static \w+: Mutex<Option<", shim + sub)) == 1 and "STAGED_KEYS" not in shim + sub
    register = re.search(r"pub fn register_committee\(.*?\n\}", shim, flags=re.S).group(0)
    assert register.count("STAGED.lock().unwrap() = None") == 2  # on success and on a failure past the argument checks
    for src, fn, kind, call in ((shim, "commit_committee", "Staged::Registration", "commit_on(c)?"),
                                (shim, "discard_committee", "Staged::Registration", "discard_on(c)?"),
                                (sub, "commit_registration", "Staged::Change", "commit_on(c)?"),
                                (sub, "discard_registration", "Staged::Change", "discard_on(c)?")):
        body = re.search(r"pub fn %s\(.*?\n\}" % fn, src, flags=re.S).group(0)
        assert "take()" not in body, fn
        assert body.index(kind) < body.index(call) < body.index("*staged = None"), fn


def test_python_forgets_a_staged_registration_the_engine_dropped():
    """A registration, update or incremental stage that succeeds leaves no staged registration in the engine, so a later commit must not
    take the staged key count."""
    from hotstuff_b200 import engine

    class Owner:
        h = None
        n_keys = 0
        _staged_keys = 777

        def _check(self, rc, what):
            assert rc == 0

    o = Owner()
    engine._committee_register(o, lambda *a: 0, "register", [[0] * 32] * 3)
    assert o._staged_keys is None and o.n_keys == 3
    for name in ("update", "stage"):
        o._staged_keys = 777
        engine._committee_update(o, lambda *a: 0, name, [[0] * 32], None)
        assert o._staged_keys is None, name
