"""Build the native pieces in-tree (nvcc for the CUDA engine, gcc for the test-only oracle / host emulation).

The product is `hotstuff_b200/libhs_crypto.so` (sm_90a only).  The oracle and the host-emulation library are test
infrastructure: building them here is not using them.
"""
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libhs_crypto.so")
ORACLE_LIB = os.path.join(ROOT, "oracle", "libhs_oracle.so")
HOSTEMU_LIB = os.path.join(ROOT, "tests", "hostemu", "libhs_hostemu.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "-shared", "-diag-suppress", "550"]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _sources(d, exts):
    return [os.path.join(d, f) for f in sorted(os.listdir(d)) if f.endswith(exts)]


def build_engine(force=False, verbose=False):
    srcs = _sources(CSRC, (".cu", ".cuh", ".cpp", ".h")) + [os.path.join(ROOT, "include", "hs_crypto.h")]
    if not force and _newer(LIB, srcs):
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, os.path.join(CSRC, "hs_engine.cu"), os.path.join(CSRC, "hs_ingest.cpp"),
                                                                                 os.path.join(CSRC, "hs_multi.cpp")]
    subprocess.check_call(cmd, cwd=ROOT)
    return LIB


def build_oracle(force=False):
    d = os.path.join(ROOT, "oracle")
    srcs = [os.path.join(d, f) for f in ("hs_oracle.c", "hs_oracle.h", "hs_constants.h")]
    if not force and _newer(ORACLE_LIB, srcs):
        return ORACLE_LIB
    subprocess.check_call(["make", "-C", d, "-B", "libhs_oracle.so"], stdout=subprocess.DEVNULL)
    return ORACLE_LIB


def build_hostemu(force=False):
    d = os.path.join(ROOT, "tests", "hostemu")
    srcs = [os.path.join(d, "hostemu.cpp")] + _sources(CSRC, (".cuh",))
    if not force and _newer(HOSTEMU_LIB, srcs):
        return HOSTEMU_LIB
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", HOSTEMU_LIB,
                           os.path.join(d, "hostemu.cpp")])
    return HOSTEMU_LIB


def build_all(force=False):
    return build_engine(force), build_oracle(force), build_hostemu(force)


if __name__ == "__main__":
    import sys
    print(build_engine(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_oracle(force="--force" in sys.argv))
    print(build_hostemu(force="--force" in sys.argv))
