"""unfilter_wave_kernel under the host SIMT emulator, against the oracle: heights that are not multiples of a band
(32 or 128 rows) and images shorter than one band, every 16-byte misalignment of the filtered rows and
of the pixels, every bpp of the fast path, one CTA working through several bands, streams that stop short of the image,
and several images in the band-level ticket order."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from test_emu_unfilter import build

POISON = 0xEE


def filtered_rows(rng, w, h, bpp, invalid_row=None):
    rows = rng.integers(0, 256, size=(h, w * bpp + 1), dtype=np.uint8)
    rows[:, 0] = rng.integers(0, 5, size=h)
    if invalid_row is not None and invalid_row < h:
        rows[invalid_row, 0] = 9      # invalid filter byte: the row passes through unchanged
    return rows.tobytes()


def run(L, filtered, w, h, bpp, depth, grid, order, shift_in=0, shift_out=0, delivered=None):
    """the kernel's pixels for `filtered` placed `shift_in` bytes and the pixels `shift_out` bytes past a 16-byte
    boundary; `delivered` bytes of the stream are usable (default: all)"""
    pitch = w * bpp
    n = len(filtered) if delivered is None else delivered
    src = (C.c_uint8 * (len(filtered) + 128))()
    base = (C.addressof(src) + 15) // 16 * 16 + shift_in
    C.memmove(base, filtered, len(filtered))
    out = (C.c_uint8 * (h * pitch + 128))(*([POISON] * (h * pitch + 128)))
    obase = (C.addressof(out) + 15) // 16 * 16 + shift_out
    L.emu_unfilter(base, n, obase, w, h, bpp, depth, grid, order)
    got = C.string_at(obase, h * pitch + 32)
    return got[: h * pitch], got[h * pitch:]


def expected(filtered, w, h, bpp, depth, rows=None):
    pitch = w * bpp
    rows = h if rows is None else rows
    if rows == 0:
        return bytes(h * pitch)
    st, px = oracle.png_unfilter(filtered[: rows * (pitch + 1)], w, rows, 8 * bpp, depth)
    assert st == 0
    return px + bytes((h - rows) * pitch)


@pytest.mark.parametrize("bpp,depth", [(1, 8), (2, 8), (3, 8), (4, 8), (6, 16), (8, 16)])
def test_heights_around_warp_and_band_sizes(bpp, depth):
    L = build()
    rng = np.random.default_rng(100 + bpp)
    for w, h in [(45, 1), (45, 31), (19, 33), (45, 127), (23, 129), (45, 200), (9, 257)]:
        f = filtered_rows(rng, w, h, bpp, invalid_row=h // 2)
        got, tail = run(L, f, w, h, bpp, depth, grid=2, order=2)
        assert got == expected(f, w, h, bpp, depth), (bpp, w, h)
        assert tail == bytes([POISON]) * len(tail)      # nothing written past the image


@pytest.mark.parametrize("shift", range(16))
def test_every_misalignment_class(shift):
    """the filtered stream and the pixels start `shift` bytes past a 16-byte boundary (rows of 4 * 37 + 1 bytes then
    start in every class anyway; the pixels' row above a band starts misaligned when the pitch is not a multiple of 16)"""
    L = build()
    rng = np.random.default_rng(shift)
    for bpp, w, h in [(4, 37, 140), (3, 50, 130)]:
        f = filtered_rows(rng, w, h, bpp)
        got, tail = run(L, f, w, h, bpp, 8, grid=2, order=shift % 4, shift_in=shift, shift_out=(5 * shift) % 16)
        assert got == expected(f, w, h, bpp, 8), (shift, bpp)
        assert tail == bytes([POISON]) * len(tail)


@pytest.mark.parametrize("order", [0, 1, 3])
def test_one_cta_takes_every_band(order):
    """a grid of one CTA, fewer warps than bands: band after band, each from the row the band before left"""
    L = build()
    rng = np.random.default_rng(40 + order)
    w, h, bpp = 70, 300, 4
    f = filtered_rows(rng, w, h, bpp, invalid_row=128)
    got, _ = run(L, f, w, h, bpp, 8, grid=1, order=order)
    assert got == expected(f, w, h, bpp, 8)


@pytest.mark.parametrize("rows", [0, 1, 100, 128, 129, 250])
def test_short_stream_leaves_missing_rows_zero(rows):
    L = build()
    rng = np.random.default_rng(7 + rows)
    w, h, bpp = 33, 260, 4
    f = filtered_rows(rng, w, h, bpp)
    got, tail = run(L, f, w, h, bpp, 8, grid=3, order=2, delivered=rows * (w * bpp + 1) + 5)
    assert got == expected(f, w, h, bpp, 8, rows), rows
    assert tail == bytes([POISON]) * len(tail)


def test_level_major_order_over_images_of_many_band_counts():
    """tickets band level by band level over images of 1 to 16 bands, fewer warps than bands in flight"""
    L = build()
    L.emu_unfilter_multi.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                     C.c_uint32, C.c_uint, C.c_int]
    rng = np.random.default_rng(11)
    bpp, depth = 4, 8
    shapes = [(21, 500), (30, 385), (17, 300), (25, 256), (40, 129), (12, 128), (33, 90), (8, 3)]   # heights descending
    filt = [filtered_rows(rng, w, h, bpp) for w, h in shapes]
    want = [expected(f, w, h, bpp, depth) for f, (w, h) in zip(filt, shapes)]
    n = len(shapes)
    for order, grid in ((0, 1), (2, 3), (5, 6)):
        srcs = [(C.c_uint8 * (len(f) + 64)).from_buffer_copy(f + bytes(64)) for f in filt]
        outs = [(C.c_uint8 * (len(px) + 64))() for px in want]
        L.emu_unfilter_multi(n, (C.c_void_p * n)(*[C.addressof(s) for s in srcs]),
                             (C.c_uint64 * n)(*[len(f) for f in filt]),
                             (C.c_void_p * n)(*[C.addressof(o) for o in outs]),
                             (C.c_uint32 * n)(*[w for w, _ in shapes]), (C.c_uint32 * n)(*[h for _, h in shapes]),
                             bpp, depth, grid, order)
        for i in range(n):
            assert bytes(outs[i])[: len(want[i])] == want[i], (i, order, grid)
            assert bytes(outs[i])[len(want[i]):] == bytes(64)
