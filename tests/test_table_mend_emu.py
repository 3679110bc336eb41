"""hs_table_mend's device steps under host emulation (tests/hostemu/table_mend_emu.cpp), CPU only.

The window findings: one wrong entry planted at each edge position of a comb table (entry 0, the anchor, entry 1 of a later window,
entry 2^(w-1) that the next window's link checks, the last entry of the last window) is always in a flagged window, and mending the
flagged windows gives back the fresh build byte for byte, storing that one entry.  The recomputation: comb_mend_block's entries equal
comb_build_block's at every key width 8..17 and the base widths 16, 20 and 24, and a correct block stores nothing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = 96


@pytest.fixture(scope="module")
def mendemu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("mendemu") / "libhs_mendemu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DHS_HOST_EMU", "-Wno-unknown-pragmas", "-o", lib,
                           os.path.join(ROOT, "tests", "hostemu", "table_mend_emu.cpp")])
    emu = ctypes.CDLL(lib)
    emu.emu_comb_table_bytes.restype = ctypes.c_uint64
    emu.emu_mend_window.restype = ctypes.c_uint64
    emu.emu_mend_block.restype = ctypes.c_uint64
    return emu


def _key(oracle, seed):
    return oracle.keygen(np.random.default_rng(seed).bytes(32))


def _table(emu, W, key):
    buf = ctypes.create_string_buffer(emu.emu_comb_table_bytes(W))
    assert emu.emu_build_comb_table(key, W, buf) == 1
    return buf


def _flags(emu, buf, W, key):
    n = emu.emu_comb_windows(W)
    out = ctypes.create_string_buffer(n + 1)
    emu.emu_mend_windows(buf, W, key, out)
    f = np.frombuffer(out.raw, np.uint8)
    return set(np.nonzero(f[:n])[0].tolist()), bool(f[n])


@pytest.mark.parametrize("W,base", [(8, False), (9, False), (10, True), (11, False)])
def test_every_edge_position_is_flagged_and_mended(mendemu, oracle, W, base):
    key = None if base else _key(oracle, W)
    clean = _table(mendemu, W, key)
    assert _flags(mendemu, clean, W, key) == (set(), False)
    n, H = mendemu.emu_comb_windows(W), 1 << (W - 1)
    stride = H + 1
    spots = [(0, 0), (0, 1), (n // 2, 1), (n // 2, H), (n - 1, H), (1, 7)]
    rng = np.random.default_rng(W)
    for win, m in spots:
        for byte in (0, int(rng.integers(1, 95)), 95):
            buf = ctypes.create_string_buffer(clean.raw, len(clean.raw))
            off = (win * stride + m) * ENTRY + byte
            buf[off] = bytes([clean.raw[off] ^ (1 << int(rng.integers(0, 8)))])
            flagged, anchor = _flags(mendemu, buf, W, key)
            assert win in flagged, (win, m, byte)
            # a failed link flags both windows it joins: the one before a wrong entry 1, the one after a wrong entry 2^(w-1)
            assert flagged <= {win - 1, win, win + 1}, (win, m, flagged)
            # the anchor reads the entry's first two coordinates; a wrong third one fails the curve equation instead
            assert anchor == ((win, m) == (0, 1) and byte < 64), (win, m, byte)
            stored = sum(mendemu.emu_mend_window(buf, W, key, w) for w in sorted(flagged))
            assert stored == 1 and buf.raw == clean.raw, (win, m, byte)
            assert _flags(mendemu, buf, W, key) == (set(), False)


def test_a_wrong_window_is_rewritten_entry_by_entry(mendemu, oracle):
    W, key = 9, _key(oracle, 1)
    clean = _table(mendemu, W, key)
    buf = ctypes.create_string_buffer(clean.raw, len(clean.raw))
    H, win = 1 << (W - 1), 3
    start = win * (H + 1) * ENTRY
    for m in (2, 3, 100, H):
        buf[start + m * ENTRY + 40] = bytes([clean.raw[start + m * ENTRY + 40] ^ 0x80])
    assert _flags(mendemu, buf, W, key)[0] == {win, win + 1}
    assert mendemu.emu_mend_window(buf, W, key, win) == 4 and mendemu.emu_mend_window(buf, W, key, win + 1) == 0
    assert buf.raw == clean.raw


@pytest.mark.parametrize("W", list(range(8, 18)) + [16, 20, 24])
def test_mend_block_equals_the_build(mendemu, oracle, W):
    rng = np.random.default_rng(100 + W)
    n, H = mendemu.emu_comb_windows(W), 1 << (W - 1)
    for key in (None, _key(oracle, 200 + W)):
        for win in (0, int(rng.integers(1, n - 1)), n - 1):
            for first in sorted({0, 64 * int(rng.integers(0, H // 64)), H - 64}):
                mended, built = ctypes.create_string_buffer(65 * ENTRY), ctypes.create_string_buffer(65 * ENTRY)
                stored = mendemu.emu_mend_block(key, W, win, first, mended, built)
                assert stored == (65 if first == 0 else 64), (W, win, first)
                assert mended.raw == built.raw, (W, win, first)
