"""The pass path of the unfilter stage (unfilter_pass_kernel, then unfilter_interleave_kernel, csrc/unfilter.cuh) under
the host SIMT emulator, against the oracle's PNG.Image.storage byte for byte: Adam7 images of every size from 1x1 to
17x17 (some passes empty), heights that give a pass 31, 32 and 33 rows, every filter distance, 1/2/4-bit images
interlaced and not, every filter type and invalid filter bytes, streams cut at every pass boundary and inside a row, and
an inflate error.  Rows are reconstructed in place, so neighbouring rows and bands hand off through the same buffer;
every case runs with the lanes in order, reversed and shuffled, and with more than one CTA."""
from __future__ import annotations

import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
import wide_rows  # noqa: E402
from oracle import oracle  # noqa: E402

ORDERS = (0, 1, 7)
TYPES = (0, 1, 2, 3, 4, 1, 4, 3, 2, 7, 4, 4, 3)   # 7: an invalid filter byte, the row stays as it is
POISON = 0xA5


def lib():
    L = emu.load("emu_unfilter_passes")
    u32p = C.POINTER(C.c_uint32)
    L.emu_unfilter_passes.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_void_p),
                                      u32p, u32p, u32p, u32p, u32p, C.POINTER(C.c_int32), C.c_uint, C.c_uint, C.c_int]
    return L


def run(images, order, grid=3, igrid=2):
    """images: [(stream, w, h, volume, depth, interlaced, status)]; the storage the pass path writes for each, checked
    for writes past its end; the streams are padded the way the library's private copies are"""
    n = len(images)
    keep, fptr, optr = [], (C.c_void_p * n)(), (C.c_void_p * n)()
    flen = (C.c_uint64 * n)()
    cols = [(C.c_uint32 * n)() for _ in range(5)]
    status = (C.c_int32 * n)()
    sizes = []
    for i, (stream, w, h, volume, depth, interlaced, st) in enumerate(images):
        src = (C.c_uint8 * (len(stream) + 64)).from_buffer_copy(bytes(stream) + bytes(64))
        size = oracle.storage_size(w, h, volume)
        # the storage starts i bytes past a 16-byte boundary: every misalignment class of the interleave's chunks
        dst = (C.c_uint8 * (size + 64))(*([POISON] * (size + 64)))
        keep += [src, dst]
        fptr[i] = C.addressof(src)
        optr[i] = (C.addressof(dst) + 15) // 16 * 16 + i % 16
        flen[i] = len(stream)
        for c, v in zip(cols, (w, h, volume, depth, int(interlaced))):
            c[i] = v
        status[i] = st
        sizes.append((size, dst))
    lib().emu_unfilter_passes(n, fptr, flen, optr, *cols, status, grid, igrid, order)
    out = []
    for i, (size, dst) in enumerate(sizes):
        base = optr[i] - C.addressof(dst)
        raw = bytes(dst)
        assert raw[:base] == bytes([POISON]) * base and raw[base + size:] == bytes([POISON]) * (len(raw) - base - size), \
            f"image {i}: written outside its storage"
        out.append(raw[base:base + size])
    return out


def expect(stream, w, h, volume, depth, interlaced, st):
    if st < 0:
        return bytes(oracle.storage_size(w, h, volume))
    return oracle.png_unfilter(bytes(stream), w, h, volume, depth, interlaced)[1]


def check(images, order, **kw):
    for im, got in zip(images, run(images, order, **kw)):
        assert got == expect(*im), im[1:]


def image(w, h, volume, depth, interlaced, seed, cut=0, types=TYPES, status=0):
    f = wide_rows.filtered_stream(w, h, volume, interlaced, types, seed)
    assert len(f) == oracle.filtered_size(w, h, volume, interlaced)
    return (bytes(f[:len(f) - cut]), w, h, volume, depth, interlaced, status)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("volume,depth", [(8, 8), (16, 8), (24, 8), (32, 8), (48, 16), (64, 16), (1, 1), (2, 2), (4, 4)])
def test_adam7_1x1_to_17x17(volume, depth, order):
    """every size from 1x1 to 17x17 in one launch (below 5x5 some passes are empty), at filter distances 1, 2, 3, 4, 6
    and 8 and at 1/2/4 bits per sample"""
    images = [image(w, h, volume, depth, True, 17 * w + h) for w in range(1, 18) for h in range(1, 18)]
    check(images, order)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("depth", [1, 2, 4])
def test_sub_byte_widths_1_to_17(depth, order):
    """1/2/4-bit rows of 1 to 17 pixels, interlaced and not: a partial last byte, and rows shorter than a chunk"""
    images = [image(w, h, depth, depth, lace, 100 * w + h + lace) for w in range(1, 18) for h in (1, 5, 40)
              for lace in (False, True)]
    check(images, order)


@pytest.mark.parametrize("order", ORDERS)
def test_passes_of_31_32_33_rows(order):
    """h = 248, 256 and 264 give pass 1 (every 8th row) 31, 32 and 33 rows, h = 257 gives passes 1 to 3 33 rows and
    passes 6 and 7 129 and 128: bands end inside a pass, at its end, and one row after it"""
    images = [image(w, h, volume, 8 if volume % 8 == 0 else volume, True, h + volume)
              for h in (248, 256, 257, 264) for w, volume in ((9, 24), (13, 8), (21, 2), (5, 64))]
    check(images, order)


@pytest.mark.parametrize("order", ORDERS)
def test_every_filter_type(order):
    """rows of one filter type each, None to Paeth and an invalid byte, and Up on the first row of every pass"""
    images = [image(37, 41, volume, 8 if volume % 8 == 0 else volume, lace, t + volume, types=(t,))
              for t in (0, 1, 2, 3, 4, 5, 255) for volume, lace in ((32, True), (24, True), (4, False), (1, True))]
    check(images, order)


@pytest.mark.parametrize("order", ORDERS)
def test_cut_streams(order):
    """streams that end at every pass boundary and one byte before and after it, in the middle of a row, and an inflate
    error: the first incomplete row ends its pass and every later one; an error reconstructs nothing"""
    images = []
    for w, h, volume, depth in ((19, 23, 32, 8), (30, 17, 1, 1), (11, 9, 48, 16)):
        full = oracle.filtered_size(w, h, volume, True)
        ends = [0]
        for _, _, sh, pitch in wide_rows.adam7_passes(w, h, volume):
            ends.append(ends[-1] + sh * (pitch + 1))
        cuts = sorted({full - e + d for e in ends for d in (-1, 0, 1) if 0 <= full - e + d <= full} |
                      {full - ends[3] - (ends[4] - ends[3]) // 2})
        images += [image(w, h, volume, depth, True, w + h, cut=c) for c in cuts]
        images.append(image(w, h, volume, depth, True, 3, status=-8))
    f = image(45, 30, 2, 2, False, 5)
    images += [image(45, 30, 2, 2, False, 5, cut=c) for c in (1, 12, 13, 14, len(f[0]) - 1)]
    check(images, order)


def test_one_cta_and_many():
    """a grid of one CTA (bands in ticket order on four warps, the interleave block by block) and more CTAs than bands"""
    images = [image(w, 70, 32, 8, True, w) for w in (3, 40, 65)]
    check(images, 2, grid=1, igrid=1)
    check(images, 3, grid=16, igrid=40)
