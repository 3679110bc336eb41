"""The audit of the verify queue's signature cache (hs_queue_sig_audit, hs_queue_sig_audit_stats, hs_scrub_sig_cache) in every binding
against include/hs_crypto.h (CPU only): the declarations and constants, the ctypes table, the Python names, the Rust submodule's extern
block and where the shim uses it, the test hook's absence from the product, and the C++ wrapper, which must compile and link."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUST_TO_C = dict(QUEUE_RUST_TO_C, **{"*mut u64": "uint64_t*"})
AUDIT_FNS = {"hs_queue_sig_audit", "hs_queue_sig_audit_stats", "hs_scrub_sig_cache"}


def test_header_declares_the_audit():
    fns = header_functions()
    assert fns["hs_queue_sig_audit"] == ("int", ["hs_queue*", "size_t", "size_t", "uint64_t*"])
    assert fns["hs_queue_sig_audit_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    assert fns["hs_scrub_sig_cache"] == ("int", ["hs_ctx*", "hs_queue*", "uint32_t"])
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_SIG_AUDIT_OUT 7\b", hdr) and re.search(r"#define HS_QUEUE_SIG_AUDIT_STATS 5\b", hdr)
    assert re.search(r"int hs_queue_sig_audit\(hs_queue \*q, size_t first_bucket, size_t n_buckets, uint64_t out\[HS_QUEUE_SIG_AUDIT_OUT\]\);", hdr)
    assert re.search(r"int hs_queue_sig_audit_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_SIG_AUDIT_STATS\]\);", hdr)
    # the new finding class takes the next bit; the scrub's counters and callback keep their layout
    assert re.search(r"#define HS_AUDIT_SIGCACHE \(1u << 5\)", hdr) and re.search(r"#define HS_AUDIT_BASE\s+\(1u << 4\)", hdr)
    assert re.search(r"#define HS_SCRUB_STATS 8\b", hdr)
    assert re.search(r"typedef void\(hs_scrub_cb\)\(void \*user, uint32_t found, uint32_t failed, size_t first_slot\);", hdr)


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib, engine
    from hotstuff_b200.engine import Engine, VerifyQueue
    u64p = ctypes.POINTER(ctypes.c_uint64)
    assert _lib.SIGNATURES["hs_queue_sig_audit"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, u64p])
    assert _lib.SIGNATURES["hs_queue_sig_audit_stats"] == (ctypes.c_int, [ctypes.c_void_p, u64p])
    assert _lib.SIGNATURES["hs_scrub_sig_cache"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32])
    assert VerifyQueue.SIG_AUDIT_OUT == ("held", "corrected", "skipped", "first_position", "first_stored", "first_derived", "first_why")
    assert VerifyQueue.SIG_AUDIT_STATS == ("audits", "checked", "corrected", "skipped", "passes")
    assert callable(VerifyQueue.sig_audit) and callable(VerifyQueue.sig_audit_stats) and callable(Engine.scrub_sig_cache)
    assert engine.AUDIT_SIGCACHE == 32


def test_rust_sig_audit_module_matches_the_header():
    src = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_sig_audit.rs")).read())
    shim = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    assert re.search(r'#\[path = "crypto_gpu_sig_audit.rs"\]\s*pub mod sig_audit;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [RUST_TO_C[r] for r in r_types] == fns[name][1], name
        assert RUST_TO_C[ret] == fns[name][0], name
        seen.add(name)
    assert seen == AUDIT_FNS
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen  # calls exactly what it declares
    assert "[0u64; 7]" in src and "[0u64; 5]" in src and "== HS_OK" in src  # HS_QUEUE_SIG_AUDIT_OUT / _STATS; a failed call is never read
    # the whole table from bucket 0 on the engine_fault branch; the scrub's slice only while the cache is on
    assert "hs_queue_sig_audit(q, 0, 0, out.as_mut_ptr())" in src
    attach = re.search(r"pub\(crate\) fn attach\(\) \{(.*?)\n\}", src, flags=re.S).group(1)
    assert attach.index("sig_cache::is_on()") < attach.index("hs_scrub_sig_cache(c, q, SIG_AUDIT_BUCKETS_PER_TICK)")


def test_rust_attaches_the_cache_to_the_scrub():
    scrub = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_scrub.rs")).read())
    start = re.search(r"pub fn start\(\) -> Result<\(\), GpuError> \{(.*?)\n\}", scrub, flags=re.S).group(1)
    assert start.index("hs_scrub_start(") < start.index("super::sig_audit::attach();")
    cache = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_sig_cache.rs")).read())
    enable = re.search(r"pub\(crate\) fn enable\(.*?\n\}", cache, flags=re.S).group(0)
    assert enable.index("ON.store(true") < enable.index("super::sig_audit::attach();")


def test_integration_snippet_audits_the_cache_on_an_engine_fault():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    branch = doc[doc.index("if xs.iter().any(|x| x.engine_fault) {"):]
    branch = branch[:branch.index("return self.verify(committee);")]
    assert "gpu::audit_tables(&committee_map)" in branch and "gpu::sig_audit::audit_cache()" in branch


def test_sig_cache_hook_is_not_in_the_product():
    from hotstuff_b200 import build
    lib = build.build_engine()
    syms = subprocess.check_output(["nm", "-D", "--defined-only", lib], text=True)
    assert re.search(r"\bhs_queue_sig_audit\b", syms) and re.search(r"\bhs_scrub_sig_cache\b", syms)
    assert not re.search(r"\bhs_test_poke_sig\b", syms)
    assert "hs_test_poke_sig" not in open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    src = open(os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")).read()
    hook = src[src.index("#ifdef HS_TEST_HOOKS"):]
    assert "extern \"C\" int hs_test_poke_sig(hs_queue *q, const uint8_t rec[128], size_t byte_offset, uint8_t xor_mask)" in hook[:hook.index("#endif")]


def test_cpp_sig_audit_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "audit.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  q.sig_cache(1 << 16);\n"
                   "  const std::array<uint64_t, HS_QUEUE_SIG_AUDIT_OUT> a = q.sig_audit();\n"
                   "  const std::array<uint64_t, HS_QUEUE_SIG_AUDIT_OUT> b = q.sig_audit(16, 32);\n"
                   "  e.scrub_sig_cache(&q, 512);\n"
                   "  e.scrub_sig_cache(nullptr);\n"
                   "  const std::array<uint64_t, HS_QUEUE_SIG_AUDIT_STATS> s = q.sig_audit_stats();\n"
                   "  return (a[1] | b[1] | s[2]) == 0 ? 0 : 1;\n"
                   "}\n")
    out = str(tmp_path / "audit")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
