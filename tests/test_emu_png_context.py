"""context_assign_kernel (online decoding: PNG.Image.assign and PNG.Image.overdraw of a range of one pass's rows,
csrc/unfilter.cuh) under the host SIMT emulator, against the oracle's PNG.Context snapshots byte for byte: every pixel
volume, row ranges that start and end at every row of every pass, widths around the kernel's 256-pixel tiles, overdraw on
and off, and the storage rows a push reports.  Lanes run in order, reversed and shuffled, on fewer CTAs than tiles."""
from __future__ import annotations

import ctypes as C
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402
from png_context_cases import (OracleContext, none_stream, random_storage, row_ends, stored_prefix,  # noqa: E402
                               stored_zlib)

ORDERS = (0, 1, 7)
POISON = 0xA5
VOLUMES = [(1, 1), (2, 2), (4, 4), (8, 8), (16, 8), (16, 16), (24, 8), (32, 8), (48, 16), (64, 16)]


def lib():
    L = emu.load("emu_png_context")
    L.emu_context_assign.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                     C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_uint, C.c_int,
                                     C.POINTER(C.c_uint64)]
    return L


def snapshot(stream, w, h, volume, depth, interlaced, k, overdraw):
    """the oracle's context after the first k filtered bytes arrived: (storage, progress)"""
    c = OracleContext(w, h, volume, depth, interlaced)
    idat = stored_zlib(stream)
    assert c.push(idat[:stored_prefix(k)], overdraw) == 0
    return c, idat


def check_range(stream, w, h, volume, depth, interlaced, ia, ib, overdraw, order, max_ctas):
    """rows ends[ia:ib] assigned by the kernel onto the oracle's storage after rows ends[:ia]: equal to the oracle's
    storage after rows ends[:ib], and the rows written equal to its progress()[4:]"""
    ends = row_ends(w, h, volume, interlaced)
    k0 = ends[ia - 1][2] if ia else 0
    c, idat = snapshot(stream, w, h, volume, depth, interlaced, k0, overdraw)
    before = c.storage()
    assert c.push(idat[stored_prefix(k0):stored_prefix(ends[ib - 1][2])], overdraw) == 0
    want, prog = c.storage(), c.progress()
    size = len(before)
    buf = (C.c_uint8 * (size + 64)).from_buffer_copy(bytes([POISON]) * 32 + before + bytes([POISON]) * 32)
    src = (C.c_uint8 * (len(stream) + 16)).from_buffer_copy(stream + bytes(16))
    lo, hi = h, 0
    for z in sorted({e[0] for e in ends[ia:ib]}):
        rows = [e[1] for e in ends[ia:ib] if e[0] == z]
        y = (C.c_uint64 * 2)()
        lib().emu_context_assign(z, rows[0], rows[-1] + 1, C.addressof(src), C.addressof(buf) + 32, w, h, volume, depth,
                                 int(interlaced), int(overdraw), max_ctas, order, y)
        lo, hi = min(lo, y[0]), max(hi, y[1])
    raw = bytes(buf)
    assert raw[:32] == bytes([POISON]) * 32 and raw[32 + size:] == bytes([POISON]) * 32, "written outside the storage"
    assert raw[32:32 + size] == want, (w, h, volume, ia, ib, overdraw)
    assert (lo, hi) == prog[4:], (prog, lo, hi)


@pytest.mark.parametrize("volume,depth", VOLUMES)
@pytest.mark.parametrize("order", ORDERS)
def test_every_range_of_a_small_adam7_image(volume, depth, order):
    """9x11 Adam7: every pair of row boundaries, overdraw on and off"""
    w, h = 9, 11
    stream = none_stream(random_storage(w, h, volume, depth, volume), w, h, volume, depth, True)
    n = len(row_ends(w, h, volume, True))
    rng = random.Random(volume * 10 + order)
    for ia in range(n):
        for ib in range(ia + 1, n + 1):
            if order and rng.random() > 0.25:   # every pair in order 0, a quarter of them in the others
                continue
            check_range(stream, w, h, volume, depth, True, ia, ib, (ia + ib) % 2 == 0, order, 2)


@pytest.mark.parametrize("w", [1, 2, 7, 8, 9, 255, 256, 257, 263])
@pytest.mark.parametrize("volume,depth", [(1, 1), (4, 4), (8, 8), (24, 8), (64, 16)])
@pytest.mark.parametrize("overdraw", [False, True])
def test_widths_around_the_tiles(w, volume, depth, overdraw):
    """rows one at a time, then the rest in one range, with few CTAs so that they stride over the tiles"""
    h = 19
    stream = none_stream(random_storage(w, h, volume, depth, w), w, h, volume, depth, True)
    n = len(row_ends(w, h, volume, True))
    order = ORDERS[w % 3]
    for ia in range(0, min(n, 24)):
        check_range(stream, w, h, volume, depth, True, ia, ia + 1, overdraw, order, 3)
    if n > 24:
        check_range(stream, w, h, volume, depth, True, 24, n, overdraw, order, 5)


@pytest.mark.parametrize("volume,depth", VOLUMES)
def test_non_interlaced(volume, depth):
    """a non-interlaced image: one pass with stride 1, nothing to paint"""
    w, h = 37, 13
    stream = none_stream(random_storage(w, h, volume, depth, 5), w, h, volume, depth, False)
    for ia, ib in ((0, 1), (1, 5), (5, 13), (0, 13)):
        check_range(stream, w, h, volume, depth, False, ia, ib, True, 7, 2)
