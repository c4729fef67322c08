"""A stream cut in two (a direct head, a symbolic tail, split_resolve_kernel, split_finish_kernel) under the host
SIMT emulator: the real kernel sources against zlib.  An accepted split must give exactly what the whole-stream
decode gives; anything else must be handed back to the whole-stream path (accept = 0) with its result untouched."""
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


@pytest.fixture(scope="module")
def lib():
    L = emu.load("emu_inflate_split")
    assert L.emu_split_result_size() == C.sizeof(emu.Result)
    L.emu_inflate_split.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.c_uint64,
                                    C.POINTER(emu.Result), C.POINTER(C.c_uint64), C.POINTER(emu.Result * 2)]
    W = emu.load("emu_inflate_wave")
    W.emu_inflate_wave.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(emu.Result), C.c_int]
    return L, W


def run_split(L, z: bytes, cap: int, share: float = 0.75, plant: int = 0, tail_cap: int = 0):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64))()
    r, at, pieces = emu.Result(), C.c_uint64(), (emu.Result * 2)()
    rc = L.emu_inflate_split(C.addressof(src), len(z), C.addressof(out), cap, share, plant, tail_cap, C.byref(r), C.byref(at),
                             C.byref(pieces))
    return rc, bytes(out)[: r.produced], r, at.value, pieces


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


@pytest.mark.parametrize("kind,w,h,share", [("photo", 640, 400, 0.75), ("photo", 333, 517, 0.55), ("graphic", 900, 700, 0.6)])
def test_head_and_tail_match_zlib(lib, kind, w, h, share):
    L, W = lib
    img = corpus.make(kind, w, h, 3)
    filt, z = corpus.zlib_png_stream(img, 4, 6)
    if kind == "graphic":
        # flat graphics fit one block: a boundary every 100 000 bytes gives the search something to find, and the
        # tail's markers then travel through long copies of copies of the head's last 32 KiB
        co = zlib.compressobj(6)
        z = b"".join(co.compress(filt[o:o + 100_000]) + co.flush(zlib.Z_SYNC_FLUSH) for o in range(0, len(filt), 100_000))
        z += co.flush()
    rc, got, r, at, pieces = run_split(L, z, len(filt), share)
    assert rc == 1, (rc, pieces[0].status, pieces[1].status)
    assert got == filt and r.checksum == zlib.adler32(filt)
    assert pieces[0].produced >= 32768 and pieces[0].consumed_bits == at and pieces[1].status == OK
    st, whole, wr = run_whole(W, z, len(filt))
    assert st == 0 and whole == got
    same_result(r, wr)


def test_noise_has_no_split_point(lib):
    """incompressible data is all stored blocks: no dynamic header to start a tail at, the stream stays whole"""
    L, _ = lib
    filt, z = corpus.zlib_png_stream(corpus.make("noise", 300, 200, 3), 4, 6)
    assert run_split(L, z, len(filt), 0.5)[0] == -1


def test_split_off_a_block_boundary_falls_back(lib):
    """a forged split point inside a block: the head runs on to the next real boundary, so the pieces cannot line up"""
    L, _ = lib
    filt, z = corpus.zlib_png_stream(corpus.make("photo", 640, 400, 3), 4, 6)
    rc, _, r, at, pieces = run_split(L, z, len(filt), plant=8 * (len(z) * 2 // 3) + 5)
    assert rc == 0 and r.status == 0 and r.produced == 0
    assert pieces[0].consumed_bits != at


def test_tail_that_overflows_its_scratch_falls_back(lib):
    L, _ = lib
    filt, z = corpus.zlib_png_stream(corpus.make("photo", 640, 400, 3), 4, 6)
    rc, _, r, _, pieces = run_split(L, z, len(filt), 0.6, tail_cap=20_000)
    assert rc == 0 and r.produced == 0 and pieces[1].status < 0


def test_truncated_and_bad_checksum_fall_back(lib):
    """both go to the whole-stream decode, which reports them exactly as an unsplit batch does"""
    L, _ = lib
    filt, z = corpus.zlib_png_stream(corpus.make("photo", 640, 400, 3), 4, 6)
    rc, _, r, _, pieces = run_split(L, z[: len(z) - 40], len(filt), 0.7)
    assert rc == 0 and r.produced == 0 and pieces[1].status != OK
    bad = bytearray(z)
    bad[-1] ^= 1
    rc, _, r, _, pieces = run_split(L, bytes(bad), len(filt), 0.7)
    assert rc == 0 and r.produced == 0 and pieces[0].status == OK and pieces[1].status == OK and pieces[1].phase == 2


def test_split_after_a_stored_block(lib):
    """incompressible data in the middle becomes stored blocks; the head crosses them, the tail's window is their end"""
    L, W = lib
    filt, _ = corpus.zlib_png_stream(corpus.make("photo", 256, 200, 4), 4, 6)
    noise = np.random.default_rng(9).integers(0, 256, 150_000, dtype=np.uint8).tobytes()
    co = zlib.compressobj(6)
    z = co.compress(filt) + co.flush(zlib.Z_SYNC_FLUSH) + co.compress(noise) + co.flush(zlib.Z_SYNC_FLUSH)
    after_stored = len(z)
    z += co.compress(filt[::-1]) + co.flush()
    plain = filt + noise + filt[::-1]
    rc, got, r, at, _ = run_split(L, z, len(plain), share=after_stored / len(z))
    assert rc == 1 and at >= 8 * after_stored and got == plain and r.checksum == zlib.adler32(plain)
    same_result(r, run_whole(W, z, len(plain))[2])
