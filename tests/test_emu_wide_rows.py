"""The scanline kernels under the host SIMT emulator on rows long enough to wrap 32-bit arithmetic (tests/wide_rows.py),
against the oracle: filter_rows_kernel on 32 MiB rows whose None score sits at 2^32, unfilter_generic_kernel on an Adam7
RGBA16 image whose pass-7 pitch is 2^29 bytes (2^32 bits), plus a small-shape sweep of unfilter_generic_kernel, and the
size functions of the C ABI at the limits geometry() accepts."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
import test_emu_filter  # noqa: E402
import wide_rows  # noqa: E402
from oracle import oracle  # noqa: E402


def test_numpy_scores_match_the_per_byte_scores():
    """wide_rows.scores, which the wide cases rely on, against test_emu_filter.scores on small random rows"""
    rng = np.random.default_rng(31)
    for bpp, n in ((1, 40), (3, 61), (4, 64), (8, 97)):
        rows = rng.integers(0, 256, size=(2, n), dtype=np.uint8)
        assert wide_rows.scores(rows[1], rows[0], bpp) == test_emu_filter.scores(bytes(rows[1]), bytes(rows[0]), bpp)


def test_filter_scores_past_2_32():
    """single 32 MiB RGBA8 rows whose None (and Up) score is 2^32 - 2048, 2^32 - 1, 2^32, 2^32 + 1 or 2^32 + 1536: the
    reference picks Sub each time, while a 32-bit sum wraps None to 0, 1 or a tie with Sub from 2^32 on and picks None"""
    cases = wide_rows.filter_cases()
    images = []
    for name, row, none in cases:
        s = wide_rows.scores(row, np.zeros_like(row), wide_rows.BPP)
        assert s[0] == s[2] == none, name
        assert wide_rows.pick(s) == 1, (name, s)
        assert wide_rows.pick(s, 32) == (0 if none >= 2 ** 32 else 1), (name, s)
        images.append((row.tobytes(), len(row) // wide_rows.BPP, 1, 32, 8, False))
    for (name, row, _), im, got in zip(cases, images, test_emu_filter.run(images)):
        want = oracle.png_filter(*im)
        assert want[0] == 1, name
        assert got[0] == want[0], f"{name}: filter {got[0]}, the reference's {want[0]}"
        assert got == want, name


def run_generic(filtered: bytearray, w, h, volume, depth, interlaced, length=None):
    L = emu.load("emu_unfilter_generic")
    L.emu_unfilter_generic.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.c_uint32]
    n = len(filtered) if length is None else length
    src = (C.c_uint8 * (len(filtered) + 64)).from_buffer(filtered + bytearray(64)) if len(filtered) < 2 ** 20 else None
    if src is None:     # wide images: no copy (the kernel reconstructs in place, the caller's buffer is spent)
        src = (C.c_uint8 * len(filtered)).from_buffer(filtered)
    size = oracle.storage_size(w, h, volume)
    out = bytearray(b"\xa5" * (size + 64))
    dst = (C.c_uint8 * len(out)).from_buffer(out)
    L.emu_unfilter_generic(C.addressof(src), n, C.addressof(dst), w, h, volume, depth, int(interlaced))
    del src, dst
    assert out[size:] == b"\xa5" * 64, "written past the image"
    del out[size:]
    return out


def check_generic(w, h, volume, depth, interlaced, types, seed, cut=0):
    filtered = wide_rows.filtered_stream(w, h, volume, interlaced, types, seed)
    assert len(filtered) == oracle.filtered_size(w, h, volume, interlaced)
    stream = bytes(filtered[:len(filtered) - cut])
    st, want = oracle.png_unfilter(stream, w, h, volume, depth, interlaced)
    assert (st != 0) == (cut > 0)     # a short stream is an error the caller reports; the pixels are still defined
    got = run_generic(bytearray(stream), w, h, volume, depth, interlaced)
    assert got == want, (w, h, volume, depth, interlaced, types, cut)


TYPES = (0, 1, 2, 3, 4, 1, 4, 3, 2)


@pytest.mark.parametrize("volume,depth", [(24, 8), (64, 16), (1, 1), (8, 8)])
def test_generic_adam7_1x1_to_9x9(volume, depth):
    """every size from 1x1 to 9x9 (below 5x5 some passes are empty), every filter type and an invalid filter byte"""
    for w in range(1, 10):
        for h in range(1, 10):
            check_generic(w, h, volume, depth, True, TYPES[(w + h) % 5:] + (7,), 100 * w + h)


@pytest.mark.parametrize("depth", [1, 2, 4])
def test_generic_sub_byte_widths_1_to_17(depth):
    """1-, 2- and 4-bit grey at every width 1..17 (the last byte of a row partly padding), non-interlaced and Adam7"""
    for w in range(1, 18):
        for h, il in ((5, False), (6, True)):
            check_generic(w, h, depth, depth, il, TYPES[w % 5:], 7 * w + depth)


def test_generic_sixteen_bit_samples():
    """16-bit grey, grey-alpha, RGB and RGBA (2, 4, 6, 8 bytes per pixel), interlaced and not"""
    for vol in (16, 32, 48, 64):
        for w, h in ((13, 7), (40, 11), (3, 3)):
            for il in (False, True):
                check_generic(w, h, vol, 16, il, TYPES[vol // 16:], vol + w)


def test_generic_short_streams_leave_rows_zero():
    """streams that end inside a row or on a row edge: the rows they do not deliver stay zero, as in the reference"""
    for w, h, vol, depth, il in ((9, 9, 32, 8, True), (17, 5, 2, 2, False), (11, 6, 64, 16, True)):
        full = oracle.filtered_size(w, h, vol, il)
        for cut in (1, (w * vol + 7) // 8 + 1, full // 2, full - 1):
            check_generic(w, h, vol, depth, il, TYPES, w * h + cut, cut)


def test_generic_adam7_pass7_pitch_2_29():
    """interlaced RGBA16 of width 2^26, two rows, Sub rows: pass 7's 2^26 pixels are 2^32 bits, so a 32-bit pitch is 0
    and the row is assigned without being reconstructed (1 GiB filtered, 1 GiB of pixels)"""
    w, h, vol = 2 ** 26, 2, 64
    filtered = wide_rows.filtered_stream(w, h, vol, True, (1,), 26)
    st, want = oracle.png_unfilter(bytes(filtered), w, h, vol, 16, True)
    assert st == 0
    got = run_generic(filtered, w, h, vol, 16, True)
    if got != want:
        bad = next(i for i in range(0, len(want), 1 << 20) if got[i:i + (1 << 20)] != want[i:i + (1 << 20)])
        first = bad + next(i for i in range(1 << 20) if got[bad + i] != want[bad + i])
        pytest.fail(f"pixels differ from byte {first} on")


def geometry_accepts(w: int, h: int, vol: int) -> bool:
    """the size rules of geometry() (csrc/pngb200_api.cu) in Python integers"""
    pitch = (w * vol + 7) // 8
    return (w < 2 ** 31 and h < 2 ** 31 and pitch <= 0xFFFFFFF0 and h * (pitch + 1) <= 2 ** 46
            and w * h * ((vol + 7) // 8) <= 2 ** 46)


# exactly at the limits: pitch 0xfffffff0 with the largest height allowed (16384), and h * (pitch + 1) == 2^46
AT_LIMITS = [(0x1FFFFFFE, 1, 64, False), (0x1FFFFFFE, 2 ** 14, 64, False), (0x1FFFFFFE, 2 ** 14, 64, True),
             (2 ** 31 - 1, 2 ** 15, 8, False), (2 ** 31 - 1, 2 ** 15, 8, True)]
INSIDE = [(2 ** 31 - 1, 7, 8, True), (2 ** 27, 3, 32, True), (2 ** 27 - 1, 2 ** 16, 64, False), (2 ** 31 - 1, 2 ** 15, 1, False)]
# one step past them, and far past (w * h * bpp near 2^62, h * (pitch + 1) near 2^49): geometry() refuses these, but the
# size functions are public and must not wrap there either
PAST_LIMITS = [(0x1FFFFFFE, 2 ** 14 + 1, 64, False), (2 ** 31 - 1, 2 ** 15 + 1, 8, False), (2 ** 31 - 1, 1, 64, False),
               (2 ** 31 - 1, 2 ** 31 - 1, 1, True), (2 ** 26, 2 ** 20, 64, True)]


@pytest.mark.parametrize("w,h,vol,il", AT_LIMITS + INSIDE + PAST_LIMITS)
def test_size_functions_at_the_geometry_limits(pngb200, w, h, vol, il):
    """pngb200_filtered_size / pngb200_storage_size against Python integers at the exact limits geometry() accepts
    (pitch 0xfffffff0 with the largest height it allows, h * (pitch + 1) == 2^46), inside them and past them: no
    product wraps"""
    assert geometry_accepts(w, h, vol) == ((w, h, vol, il) not in PAST_LIMITS)
    assert pngb200.filtered_size(w, h, vol, il) == wide_rows.filtered_size(w, h, vol, il)
    assert pngb200.storage_size(w, h, vol) == w * h * ((vol + 7) // 8)
