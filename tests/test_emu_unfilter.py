"""unfilter_wave_kernel (csrc/unfilter.cuh) under the host SIMT emulator, built exactly as the library builds it: every
filter type, ragged widths, misaligned rows, several bands talking through the progress words, against the oracle."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

HERE = os.path.join(os.path.dirname(__file__), "emu")


def build():
    lib = os.path.join(HERE, "libemu_unfilter.so")
    src = os.path.join(HERE, "emu_unfilter.cpp")
    dep = os.path.join(HERE, "..", "..", "swift-png_b200", "csrc", "unfilter.cuh")
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in (src, dep, os.path.join(HERE, "simt.h"))):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-shared", "-fPIC", "-I" + HERE, "-Wno-attributes",
                        "-o", lib, src], check=True)
    L = C.CDLL(lib)
    L.emu_unfilter.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint, C.c_int]
    return L


# (scheduling order, CTAs): grid 1 holds 4 warps, fewer than the 7 bands of the 200-row shapes, so warps take later tickets
@pytest.mark.parametrize("order,grid", [(0, 2), (1, 1), (2, 4), (3, 3)])
def test_wave_kernel_matches_oracle(order, grid):
    L = build()
    rng = np.random.default_rng(14)
    for bpp, depth, w, h in [(4, 8, 300, 100), (4, 8, 37, 70), (8, 16, 129, 67), (3, 8, 211, 40), (1, 8, 1000, 33),
                             (4, 8, 3, 200), (2, 8, 64, 64), (6, 16, 50, 97), (4, 8, 1024, 64)]:
        pitch = w * bpp
        rows = rng.integers(0, 256, size=(h, pitch + 1), dtype=np.uint8)
        rows[:, 0] = rng.integers(0, 5, size=h)
        if h > 40:
            rows[37, 0] = 7     # invalid filter byte: the row passes through unchanged
        filtered = rows.tobytes()
        st, want = oracle.png_unfilter(filtered, w, h, 8 * bpp, depth)
        assert st == 0
        src = (C.c_uint8 * (len(filtered) + 64)).from_buffer_copy(filtered + bytes(64))
        out = (C.c_uint8 * (h * pitch + 64))()
        L.emu_unfilter(C.addressof(src), len(filtered), C.addressof(out), w, h, bpp, depth, grid, order)
        assert bytes(out)[: h * pitch] == want, (bpp, depth, w, h, order)
        assert bytes(out)[h * pitch:] == bytes(64)      # nothing written past the image


def test_level_major_ticket_order_over_several_images():
    """tickets handed out band level by band level over images of different heights (run_unfilter's order): every band still
    finds the band above it running, every image comes out as the oracle's"""
    L = build()
    L.emu_unfilter_multi.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                     C.c_uint, C.c_int]
    rng = np.random.default_rng(5)
    bpp, depth = 4, 8
    shapes = [(90, 200), (40, 130), (200, 130), (33, 64), (64, 31), (17, 5)]      # (w, h), heights descending
    filt, want, srcs, outs = [], [], [], []
    for w, h in shapes:
        rows = rng.integers(0, 256, size=(h, w * bpp + 1), dtype=np.uint8)
        rows[:, 0] = rng.integers(0, 5, size=h)
        f = rows.tobytes()
        st, px = oracle.png_unfilter(f, w, h, 8 * bpp, depth)
        assert st == 0
        filt.append(f)
        want.append(px)
    for order, grid in ((0, 2), (2, 3), (1, 4)):
        srcs = [(C.c_uint8 * (len(f) + 64)).from_buffer_copy(f + bytes(64)) for f in filt]
        outs = [(C.c_uint8 * (len(px) + 64))() for px in want]
        n = len(shapes)
        fp = (C.c_void_p * n)(*[C.addressof(s_) for s_ in srcs])
        fl = (C.c_uint64 * n)(*[len(f) for f in filt])
        op = (C.c_void_p * n)(*[C.addressof(o) for o in outs])
        ws = (C.c_uint32 * n)(*[w for w, _ in shapes])
        hs = (C.c_uint32 * n)(*[h for _, h in shapes])
        L.emu_unfilter_multi(n, fp, fl, op, ws, hs, bpp, depth, grid, order)
        for i in range(n):
            assert bytes(outs[i])[: len(want[i])] == want[i], (i, order)
