"""A split stream's tail that leaves symbolic mode (StreamJob.may_switch): once the last 32 KiB it produced hold no
marker, it goes on in bytes behind its symbols, and split_resolve_kernel copies those bytes behind the head's.  The
real kernel sources under the host SIMT emulator, against zlib and the whole-stream decode."""
from __future__ import annotations

import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import corpus  # noqa: E402
import emu  # noqa: E402

ZLIB = 0
OK = 0
ERR_OUTPUT_CAPACITY = -64


@pytest.fixture(scope="module")
def lib():
    L = emu.load("emu_inflate_switch")
    assert L.emu_switch_result_size() == C.sizeof(emu.Result)
    L.emu_inflate_switch.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.c_uint64,
                                     C.c_uint32, C.POINTER(emu.Result), C.POINTER(C.c_uint64), C.POINTER(emu.Result * 2),
                                     C.POINTER(C.c_uint64 * 2)]
    W = emu.load("emu_inflate_wave")
    W.emu_inflate_wave.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(emu.Result), C.c_int]
    return L, W


def run_split(L, z: bytes, cap: int, share: float = 0.5, plant: int = 0, tail_cap: int = 0, may_switch: int = 1):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64))()
    r, at, pieces, sw = emu.Result(), C.c_uint64(), (emu.Result * 2)(), (C.c_uint64 * 2)()
    rc = L.emu_inflate_switch(C.addressof(src), len(z), C.addressof(out), cap, share, plant, tail_cap, may_switch,
                              C.byref(r), C.byref(at), C.byref(pieces), C.byref(sw))
    return rc, bytes(out)[: r.produced], r, at.value, pieces, (sw[0], sw[1])


def run_whole(W, z: bytes, cap: int):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64))()
    r = emu.Result()
    st = W.emu_inflate_wave(C.addressof(src), len(z), C.addressof(out), cap, ZLIB, C.byref(r), 0)
    return st, bytes(out)[: r.produced], r


def same_result(a: emu.Result, b: emu.Result):
    for f in ("status", "err_a", "err_b", "checksum", "blocks", "declared", "produced", "consumed_bits", "resume_bit",
              "resume_out", "trailer_seen", "phase", "ck_done"):
        assert getattr(a, f) == getattr(b, f), f


def narrow_photo():
    """narrow and tall: 32 KiB spans few rows, so the markers of the tail's first rows die out early in the tail"""
    filt, z = corpus.zlib_png_stream(corpus.make("photo", 96, 3000, 5), 4, 6)
    return filt, z


def check_against_whole(W, z, plain, rc, got, r):
    assert rc == 1
    assert got == plain and r.checksum == zlib.adler32(plain)
    st, whole, wr = run_whole(W, z, len(plain))
    assert st == 0 and whole == got
    same_result(r, wr)


def test_photo_tail_switches(lib):
    L, W = lib
    filt, z = narrow_photo()
    rc, got, r, at, pieces, (m, area) = run_split(L, z, len(filt), 0.5)
    assert 0 < m < pieces[1].produced, (m, pieces[1].produced)
    assert area % 16 == 0 and area >= 2 * m + 32768
    check_against_whole(W, z, filt, rc, got, r)
    # the same tail without the switch: all symbols, no switch record, same result
    rc2, got2, r2, _, pieces2, sw2 = run_split(L, z, len(filt), 0.5, may_switch=0)
    assert sw2 == (0, 0) and pieces2[1].produced == pieces[1].produced
    assert rc2 == 1 and got2 == got
    same_result(r2, r)


def test_graphic_tail_never_switches(lib):
    """copies of copies of the head's last 32 KiB: the markers never die out, the tail stays symbolic (m = n2)"""
    L, W = lib
    filt, _ = corpus.zlib_png_stream(corpus.make("graphic", 900, 700, 3), 4, 6)
    co = zlib.compressobj(6)
    z = b"".join(co.compress(filt[o:o + 100_000]) + co.flush(zlib.Z_SYNC_FLUSH) for o in range(0, len(filt), 100_000))
    z += co.flush()
    rc, got, r, _, pieces, (m, _) = run_split(L, z, len(filt), 0.6)
    assert m == pieces[1].produced > 0
    check_against_whole(W, z, filt, rc, got, r)


def fresh_block_then(next_part: str):
    """head, then (after a full flush, so nothing refers back across it) one dynamic block of 33 000 bytes that is
    clean once it ends, then a stored block and a final block, or the final block right away"""
    rows, _ = corpus.zlib_png_stream(corpus.make("photo", 256, 160, 7), 4, 6)
    head, clean, rest = rows[:60_000], rows[60_000:93_000], rows[93_000:]
    noise = np.random.default_rng(11).integers(0, 256, 70_000, dtype=np.uint8).tobytes()
    co = zlib.compressobj(6)
    z = co.compress(head) + co.flush(zlib.Z_FULL_FLUSH)
    at = 8 * len(z)
    z += co.compress(clean) + co.flush(zlib.Z_FULL_FLUSH)
    if next_part == "stored":
        z += co.compress(noise) + co.flush(zlib.Z_SYNC_FLUSH)
        plain = head + clean + noise + rest
    else:
        plain = head + clean + rest
    z += co.compress(rest) + co.flush()
    return z, plain, at, len(clean)


@pytest.mark.parametrize("next_part", ["stored", "final"])
def test_switch_right_before_a_block(lib, next_part):
    L, W = lib
    z, plain, at, m = fresh_block_then(next_part)
    rc, got, r, _, pieces, (sw_out, _) = run_split(L, z, len(plain), plant=at)
    assert sw_out == m < pieces[1].produced
    check_against_whole(W, z, plain, rc, got, r)


def test_byte_area_overflow_falls_back(lib):
    L, _ = lib
    filt, z = narrow_photo()
    _, _, _, _, pieces, (m, _) = run_split(L, z, len(filt), 0.5)
    n2 = pieces[1].produced
    # room for the symbols and the window, half the bytes behind them
    rc, _, r, _, pieces, (m2, _) = run_split(L, z, len(filt), 0.5, tail_cap=m + 16_400 + (n2 - m) // 4)
    assert rc == 0 and r.produced == 0 and r.status == 0
    assert pieces[1].status == ERR_OUTPUT_CAPACITY and 0 < m2 < n2


def test_truncated_and_bad_checksum_after_the_switch_fall_back(lib):
    L, _ = lib
    filt, z = narrow_photo()
    rc, _, r, _, pieces, (m, _) = run_split(L, z[: len(z) - 40], len(filt), 0.5)
    assert rc == 0 and r.produced == 0 and pieces[1].status != OK
    assert 0 < m < pieces[1].produced
    bad = bytearray(z)
    bad[-1] ^= 1
    rc, _, r, _, pieces, (m, _) = run_split(L, bytes(bad), len(filt), 0.5)
    assert rc == 0 and r.produced == 0 and pieces[0].status == OK and pieces[1].status == OK and pieces[1].phase == 2
    assert 0 < m < pieces[1].produced
