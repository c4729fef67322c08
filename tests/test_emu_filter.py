"""filter_rows_kernel (csrc/filter.cuh) under the host SIMT emulator against oracle.png_filter: exact score ties between
neighbouring filters, sub-byte depths at every width up to 17, Adam7 with empty passes, 16-bit samples, and batches whose
image boundaries fall on CTA boundaries (8 rows per CTA)."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

FILTER_WARPS = 8
SHUFFLED = 5


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def scores(cur: bytes, prev: bytes, bpp: int):
    """the five sum|int8| scores of PNG.Encoder.score for one row (None, Sub, Up, Average, Paeth)"""
    s = [0] * 5
    for i, x in enumerate(cur):
        a = cur[i - bpp] if i >= bpp else 0
        b = prev[i]
        c = prev[i - bpp] if i >= bpp else 0
        for k, p in enumerate((0, a, b, (a + b) >> 1, paeth(a, b, c))):
            v = (x - p) & 0xFF
            s[k] += 256 - v if v & 0x80 else v
    return s


def run(images, order=0):
    """images: [(storage, w, h, volume, depth, interlaced)] -> filtered streams from one emulated launch"""
    L = emu.load("emu_filter")
    n = len(images)
    srcs, dsts = [], []
    for st, w, h, vol, depth, il in images:
        srcs.append((C.c_uint8 * max(len(st), 1)).from_buffer_copy(st or b"\0"))
        dsts.append((C.c_uint8 * (oracle.filtered_size(w, h, vol, il) + 64)).from_buffer_copy(
            b"\xa5" * (oracle.filtered_size(w, h, vol, il) + 64)))
    ptrs = lambda bufs: (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    u32 = lambda i: (C.c_uint32 * n)(*[im[i] for im in images])
    u8 = lambda i: (C.c_uint8 * n)(*[int(im[i]) for im in images])
    L.emu_filter_batch(n, ptrs(srcs), ptrs(dsts), u32(1), u32(2), u8(3), u8(4), u8(5), order)
    out = []
    for d, (st, w, h, vol, depth, il) in zip(dsts, images):
        size = oracle.filtered_size(w, h, vol, il)
        raw = bytes(d)
        assert raw[size:] == b"\xa5" * 64, "written past the filtered stream"
        out.append(raw[:size])
    return out


def check(images, order=0):
    for im, got in zip(images, run(images, order)):
        st, w, h, vol, depth, il = im
        assert got == oracle.png_filter(st, w, h, vol, depth, il), (w, h, vol, depth, il, order)


def image(rng, w, h, vol, depth, il=False, hi=None):
    bpp = (vol + 7) >> 3
    top = (1 << depth) if depth < 8 else 256
    return (rng.integers(0, hi or top, w * h * bpp, dtype=np.uint8).tobytes(), w, h, vol, depth, il)


def tie_rows(rng, first: int, second: int, w: int = 6):
    """a two-row grey image whose second row scores filters `first` and `second` equal and lowest"""
    for _ in range(200000):
        rows = rng.integers(0, 12, size=(2, w), dtype=np.uint8)
        s = scores(bytes(rows[1]), bytes(rows[0]), 1)
        if s[first] == s[second] == min(s) and s.index(min(s)) == first:
            return rows.tobytes()
    raise AssertionError("no tie found")


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_ties_pick_the_first_filter(orc, order):
    """rows where None/Sub, Sub/Up, Up/Average and Average/Paeth tie exactly: the earlier filter wins (strict <, as in
    PNG.Encoder.filter); an all-zero image (every score 0) and bytes of 0x80 (score 128 each)"""
    rng = np.random.default_rng(21)
    images = []
    for first, second in ((0, 1), (1, 2), (2, 3), (3, 4)):
        data = tie_rows(rng, first, second)
        images.append((data, 6, 2, 8, 8, False))
        got = oracle.png_filter(data, 6, 2, 8, 8)
        assert got[7] == first      # the second row's filter byte
    images += [(bytes(40 * 9 * 4), 40, 9, 32, 8, False), (b"\x80" * 33 * 5, 33, 5, 8, 8, False),
               (b"\x80" * 17 * 17 * 2, 17, 17, 16, 8, True)]
    check(images, order)


@pytest.mark.parametrize("volume", [1, 2, 4])
def test_sub_byte_widths_1_to_17(orc, volume):
    """1-, 2- and 4-bit samples (grey or palette indices: the filter sees the same bytes) at every width 1..17, with the
    rest of the last byte of a row zero; non-interlaced and Adam7"""
    rng = np.random.default_rng(volume)
    images = [image(rng, w, h, volume, volume, il) for w in range(1, 18) for h, il in ((3, False), (6, True))]
    check(images)


def test_adam7_with_empty_passes(orc):
    """every size from 1x1 to 9x9, 8-bit RGB and 1-bit grey: below 5x5 some of the seven passes are empty"""
    rng = np.random.default_rng(7)
    images = [image(rng, w, h, vol, depth, True) for w in range(1, 10) for h in range(1, 10)
              for vol, depth in ((24, 8), (1, 1)) if (w + h + vol) % 2 == 0 or w == h]
    check(images)


@pytest.mark.parametrize("order", [0, SHUFFLED])
def test_sixteen_bit_samples(orc, order):
    """16-bit grey-alpha (4 bytes per pixel) and RGBA (8), interlaced and not"""
    rng = np.random.default_rng(16)
    images = [image(rng, w, h, vol, 16, il) for vol in (32, 64) for (w, h) in ((13, 7), (40, 11), (3, 3)) for il in (False, True)]
    images.append(image(rng, 70, 9, 64, 16, False, hi=8))    # small differences: the filters' scores are close
    check(images, order)


def test_batch_row_bases_on_cta_edges(orc):
    """images of 8, 16, 7, 9 and 1 rows back to back (row_base lands on and next to the 8-row CTA edges), mixing
    interlaced and non-interlaced images and several pixel formats in one launch"""
    rng = np.random.default_rng(3)
    images = [image(rng, 20, 8, 32, 8), image(rng, 5, 16, 24, 8), image(rng, 9, 7, 8, 8, True), image(rng, 30, 9, 2, 2),
              image(rng, 64, 1, 64, 16), image(rng, 11, 8, 16, 16, True), image(rng, 1, 1, 8, 8), image(rng, 33, 24, 4, 4)]
    check(images)
    check(images[::-1], 1)
