"""The verify queue's explain lane (hs_queue_explain, hs_queue_submit_explain, hs_queue_submit_explain_msgs, hs_queue_explain_stats) in
every binding against include/hs_crypto.h (CPU only): the declarations, the ctypes table, the Python names, the Rust submodule's extern
block and its status handling, the C++ wrapper (which must compile and link), and the kernel's one launch site, whose launcher passes no
context table."""
import ctypes
import os
import re
import subprocess

from test_binding_consistency import _strip_comments, header_functions
from test_launch_sites import LAUNCH, _code
from test_queue_bindings import QUEUE_RUST_TO_C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPLAIN_SIG = ("int", ["hs_queue*", "const hs_rec128*", "size_t", "hs_queue_cb*", "void*", "size_t*"])
EXPLAIN_MSGS_SIG = ("int", ["hs_queue*", "const uint8_t*", "const uint64_t*", "size_t", "const uint8_t*", "const uint8_t*", "const uint32_t*",
                            "size_t", "hs_queue_cb*", "void*", "size_t*"])
RUST = os.path.join(ROOT, "rust", "crypto_gpu_explain_queue.rs")


def test_header_declares_the_explain_lane():
    fns = header_functions()
    assert fns["hs_queue_explain"] == ("int", ["hs_queue*", "size_t", "size_t"])
    assert fns["hs_queue_submit_explain"] == EXPLAIN_SIG
    assert fns["hs_queue_submit_explain_msgs"] == EXPLAIN_MSGS_SIG
    assert fns["hs_queue_explain_stats"] == ("int", ["hs_queue*", "uint64_t*"])
    # the msgs form takes hs_queue_submit_msgs' arrays, without the modes
    msgs = fns["hs_queue_submit_msgs"][1]
    assert EXPLAIN_MSGS_SIG[1] == msgs[:7] + msgs[8:]
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "hs_crypto.h")).read())
    assert re.search(r"#define HS_QUEUE_EXPLAIN_STATS 3\b", hdr)
    assert re.search(r"int hs_queue_explain_stats\(hs_queue \*q, uint64_t out\[HS_QUEUE_EXPLAIN_STATS\]\);", hdr)
    # the existing counters keep their layouts
    assert re.search(r"#define HS_QUEUE_STATS 6\b", hdr) and re.search(r"#define HS_QUEUE_BATCH_STATS 5\b", hdr)
    assert re.search(r"#define HS_QUEUE_GENERIC_STATS 3\b", hdr) and re.search(r"#define HS_QUEUE_DIGEST_STATS 4\b", hdr)


def test_ctypes_and_python_names():
    from hotstuff_b200 import _lib
    from hotstuff_b200.engine import VerifyQueue
    P = ctypes.POINTER
    assert _lib.SIGNATURES["hs_queue_explain"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t])
    assert _lib.SIGNATURES["hs_queue_submit_explain"] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                                                         ctypes.c_void_p, P(ctypes.c_size_t)])
    ret, args = _lib.SIGNATURES["hs_queue_submit_explain_msgs"]
    assert ret is ctypes.c_int and len(args) == len(EXPLAIN_MSGS_SIG[1])
    assert args[3] is ctypes.c_size_t and args[7] is ctypes.c_size_t and args[10] == P(ctypes.c_size_t)
    assert all(a is ctypes.c_void_p for k, a in enumerate(args[:10]) if k not in (3, 7))
    assert _lib.SIGNATURES["hs_queue_explain_stats"] == (ctypes.c_int, [ctypes.c_void_p, P(ctypes.c_uint64)])
    assert VerifyQueue.EXPLAIN_STATS == ("launches", "records", "requests")
    for name in ("explain", "submit_explain", "submit_explain_msgs", "explain_stats"):
        assert callable(getattr(VerifyQueue, name)), name


def test_python_reads_an_explain_ticket_as_packed_bytes():
    import numpy as np
    from hotstuff_b200.engine import VerifyQueue, _WhyCount
    for n in (1, 3, 4, 5, 9):
        why = np.arange(1, n + 1, dtype=np.uint8)
        words = np.zeros(VerifyQueue._n_words(_WhyCount(n)), np.uint32)
        assert len(words) == (n + 3) // 4
        words.view(np.uint8)[:n] = why  # byte i of the little-endian packing is record i
        assert (VerifyQueue._bools(words, _WhyCount(n)) == why).all()
    assert VerifyQueue._n_words(5) == 1 and VerifyQueue._n_words((3, 40)) == 3  # record counts and batch tickets keep their layouts


def test_rust_explain_module_matches_the_header():
    src = _strip_comments(open(RUST).read())
    shim = open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read()
    assert re.search(r'#\[path = "crypto_gpu_explain_queue.rs"\]\s*pub mod explain_queue;', shim)
    block = re.search(r'extern\s+"C"\s*\{(.*?)\n\}', src, flags=re.S).group(1)
    fns = header_functions()
    rust_to_c = dict(QUEUE_RUST_TO_C, **{"*const HsRec128": "const hs_rec128*"})
    seen = set()
    for m in re.finditer(r"fn\s+(hs_\w+)\s*\((.*?)\)\s*(?:->\s*([^;]+))?;", block, flags=re.S):
        name, params, ret = m.group(1), m.group(2), (m.group(3) or "").strip()
        r_types = [re.sub(r"\s+", " ", p.split(":", 1)[1].strip()) for p in params.split(",") if p.strip()]
        assert [rust_to_c[r] for r in r_types] == fns[name][1], name
        assert rust_to_c[ret] == fns[name][0], name
        seen.add(name)
    assert seen == {"hs_queue_explain", "hs_queue_submit_explain"}
    assert set(re.findall(r"\b(hs_\w+)\s*\(", src.replace(block, ""))) == seen
    assert re.search(r"use super::queue::\{[^}]*\bqueue\b[^}]*\bHsQueueCb\b[^}]*\};", src)
    on_done = re.search(r"unsafe extern \"C\" fn on_done\((.*?)\)", src).group(1)
    assert [QUEUE_RUST_TO_C[p.split(":", 1)[1].strip()] for p in on_done.split(",")] == ["void*", "size_t", "int", "const uint32_t*"]


def test_rust_helper_submits_every_rejected_record_in_one_request_and_maps_a_refusal_to_none():
    src = _strip_comments(open(RUST).read())
    fn = re.search(r"pub async fn explain_rejected_queued\(recs: &\[HsRec128\], modes: &\[u8\], verdicts: &\[bool\]\) -> Option<Vec<Explained>> \{"
                   r"(.*?)\n\}", src, flags=re.S).group(1)
    # every rejected record, in record order, goes into one request
    assert "let index: Vec<usize> = (0..recs.len()).filter(|&i| !verdicts[i]).collect();" in fn
    assert "let rejected: Vec<HsRec128> = index.iter().map(|&i| recs[i]).collect();" in fn
    assert len(re.findall(r"\bhs_queue_submit_explain\(", fn)) == 1
    assert "hs_queue_submit_explain(q, rejected.as_ptr(), rejected.len(), Some(on_done), user, std::ptr::null_mut())" in fn
    assert not re.search(r"\b(for|while|loop)\b", fn.split("let rx", 1)[1].split("rx.await", 1)[0])  # no retry, no second request
    # a refusal is None and frees the pending state; an engine failure is None; the lane is turned on once, and only HS_OK counts
    assert re.search(r"if rc != HS_OK \{\s*drop\(unsafe \{ Box::from_raw\(user as \*mut Pending\) \}\);\s*return None;", fn)
    assert "if !enable(q, EXPLAIN_MAX_RECORDS, EXPLAIN_MAX_BYTES) { return None; }" in fn
    assert "let why = rx.await.ok().flatten()?;" in fn
    on_done = re.search(r"unsafe extern \"C\" fn on_done\(.*?\n\}", src, flags=re.S).group(0)
    assert re.search(r"let out = if status == HS_OK \{.*?\} else \{\s*None\s*\};", on_done, flags=re.S)
    assert "(*bitmap.add(i / 4) >> (8 * (i % 4))) as u8" in on_done  # the packed bytes, little-endian
    enable = re.search(r"pub\(crate\) fn enable\(.*?\n\}", src, flags=re.S).group(0)
    assert "call_once" in enable and "hs_queue_explain(q, max_records, max_bytes) } == HS_OK" in enable
    # engine_fault exactly as explain_rejected sets it: the record is valid in its own mode
    assert "why & !(HS_WHY_A_SMALL | HS_WHY_R_SMALL) == 0" in fn and "why == 0" in fn
    assert "Explained { index: i, why, engine_fault: valid }" in fn
    shim = _strip_comments(open(os.path.join(ROOT, "rust", "crypto_gpu_shim.rs")).read())
    assert "pub fn explain_rejected(recs: &[HsRec128], modes: &[u8], verdicts: &[bool]) -> Option<Explained>" in shim


def test_k_queue_explain_has_one_launch_site_and_its_launcher_passes_no_table():
    code = _code()
    launches = [m.group(1) for m in LAUNCH.finditer(code)]
    assert launches.count("k_queue_explain") == 1
    launcher = re.search(r"static cudaError_t launch_queue_explain\(.*?\n\}", code, flags=re.S).group(0)
    assert "k_queue_explain<<<" in launcher and "c->launches++" in launcher
    for table in ("atables", "d_btable", "keys.", "slots", "committee_tables", "ctx_tables", "comb_params"):
        assert table not in launcher, table
    # the kernel's parameters are the request list, the counts and the lane's two buffers: no table type
    params = re.search(r"k_queue_explain\((.*?)\)\s*\{", code, flags=re.S).group(1)
    for table in ("ge_niels", "committee_tables", "comb_params", "sig_cache_dev", "small_rec"):
        assert table not in params, table
    # the only caller is the lane's dispatch
    assert len(re.findall(r"\blaunch_queue_explain\(", code)) == 2


def test_cpp_explain_compiles_and_links(tmp_path):
    from hotstuff_b200 import build
    lib = build.build_engine()
    src = tmp_path / "explain.cpp"
    src.write_text('#include "hs_crypto.hpp"\n'
                   "int main(int argc, char **) {\n"
                   "  if (argc < 2) return 0;  // linked, not run\n"
                   "  hs::Engine e(0);\n"
                   "  hs::VerifyQueue q(e, 1024);\n"
                   "  q.explain(1024, 1 << 20);\n"
                   "  hs_rec128 r[2] = {};\n"
                   "  const uint8_t pre[16] = {};\n"
                   "  const uint64_t off[2] = {0, 16};\n"
                   "  uint8_t sig[2 * 64] = {}, pk[2 * 32] = {};\n"
                   "  const uint32_t idx[2] = {0, 0};\n"
                   "  try {\n"
                   "    const std::vector<uint8_t> a = q.submit_explain(r, 2).get();\n"
                   "    const std::vector<uint8_t> b = q.submit_explain_msgs(pre, off, 1, sig, pk, idx, 2).get();\n"
                   "    const std::array<uint64_t, HS_QUEUE_EXPLAIN_STATS> s = q.explain_stats();\n"
                   "    return a.size() == 2 && b.size() == 2 && s[2] == 2 ? 0 : 1;\n"
                   "  } catch (const hs::QueueFull &) {\n"
                   "    return 2;\n"
                   "  }\n"
                   "}\n")
    out = str(tmp_path / "explain")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", out, str(src), lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    assert os.path.exists(out)
