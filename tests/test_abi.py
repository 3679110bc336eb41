"""The C-ABI library loads and exports every symbol include/hs_crypto.h declares (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "hs_crypto.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(hs_[a-z0-9_]+)\s*\(", hdr)))


def test_library_builds_and_exports_every_declared_symbol():
    from hotstuff_b200 import build, _lib
    path = build.build_engine()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    syms = declared_symbols()
    assert len(syms) >= 17
    for s in syms:
        assert hasattr(lib, s), "missing export %s" % s
    assert sorted(_lib.SIGNATURES) == syms, "python binding table out of sync with the header"
    _lib.load()


def test_library_is_sm90a_only():
    from hotstuff_b200 import build
    import subprocess
    out = subprocess.run(["cuobjdump", "--list-elf", build.build_engine()], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from hotstuff_b200 import Engine, EngineError
    with pytest.raises(EngineError):
        Engine(0)


def test_product_does_not_touch_the_oracle():
    """The shipped package must not import / link / dlopen anything under oracle/ or tests/."""
    pkg = os.path.join(ROOT, "hotstuff_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")) and f != "build.py":
                txt = open(os.path.join(dirpath, f)).read()
                assert "hs_oracle" not in txt and "libhs_oracle" not in txt and "hostemu.cpp" not in txt, os.path.join(dirpath, f)
