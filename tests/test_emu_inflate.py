"""inflate_wave_kernel under the host SIMT emulator (tests/emu): the kernel's control flow -- chain walk,
ring window, deferred copies, Adler-32 folding, fallbacks -- against zlib and the oracle, without a GPU.
The emulator runs one fiber per CUDA thread; three scheduling orders shake out order dependence between
barriers.  (The GPU tests in test_gpu_decode.py run the same kernel on hardware.)"""
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
from oracle import oracle  # noqa: E402

ZLIB, RAW, GZIP = 0, 1, 2   # pngb200_format: zlib, ios (raw deflate), gzip


@pytest.fixture(scope="module")
def lib():
    L = emu.load("emu_inflate_wave")
    assert L.emu_result_size() == C.sizeof(emu.Result)
    L.emu_inflate_wave.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(emu.Result), C.c_int]
    return L


def run(L, z: bytes, cap: int, fmt: int = ZLIB, order: int = 0, misalign: int = 0):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64 + misalign))()
    r = emu.Result()
    st = L.emu_inflate_wave(C.addressof(src), len(z), C.addressof(out) + misalign, cap, fmt, C.byref(r), order)
    return st, bytes(out)[misalign:misalign + r.produced], r


def photo_stream(w, h, level=6, seed=0):
    img = corpus.make("photo", w, h, seed)
    return corpus.zlib_png_stream(img, 4, level)


@pytest.mark.parametrize("order", [0, 1, 5])
def test_photo_all_orders(lib, order):
    filt, z = photo_stream(320, 200)
    st, got, r = run(lib, z, len(filt), order=order)
    assert st == 0 and got == filt
    assert r.ck_done == 1 and r.checksum == zlib.adler32(filt) and r.stat[3] == 0


@pytest.mark.parametrize("kind,w,h", [("graphic", 640, 480), ("noise", 128, 64), ("photo", 97, 33)])
def test_corpora(lib, kind, w, h):
    img = corpus.make(kind, w, h, 1)
    filt, z = corpus.zlib_png_stream(img, 4, 6)
    for mis in (0, 5):
        st, got, r = run(lib, z, len(filt), misalign=mis)
        assert st == 0 and got == filt and r.checksum == zlib.adler32(filt) and r.stat[3] == 0


def test_levels_and_strategies(lib):
    filt, _ = photo_stream(256, 96)
    for level in (1, 4, 9):
        z = zlib.compress(filt, level)
        st, got, r = run(lib, z, len(filt))
        assert st == 0 and got == filt
    for strategy in (zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE):
        co = zlib.compressobj(6, zlib.DEFLATED, 15, 9, strategy)
        z = co.compress(filt) + co.flush()
        st, got, r = run(lib, z, len(filt))
        assert st == 0 and got == filt and r.checksum == zlib.adler32(filt), strategy


def test_mixed_blocks_ring_refill(lib):
    """stored blocks, oversized waves (flat data) and ordinary waves in one stream: the ring has to be
    refilled from HBM whenever bytes were written behind its back"""
    rng = np.random.default_rng(7)
    filt, _ = photo_stream(256, 64)
    parts = [filt, bytes(200_000), rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes(), filt[::-1],
             b"ab" * 150_000, filt]
    co = zlib.compressobj(6)
    z = b""
    for i, p in enumerate(parts):
        z += co.compress(p)
        z += co.flush(zlib.Z_FULL_FLUSH if i % 2 else zlib.Z_SYNC_FLUSH)
    z += co.flush()
    plain = b"".join(parts)
    for order in (0, 3):
        st, got, r = run(lib, z, len(plain), order=order)
        assert st == 0 and got == plain and r.checksum == zlib.adler32(plain) and r.stat[3] == 0


def test_reference_encoder_stream(lib):
    """a stream as the reference's own encoder writes it (level 9: one growing dynamic block per 2^k bytes)"""
    filt, _ = photo_stream(200, 120)
    z = oracle.deflate(filt, 9)
    st, got, r = run(lib, z, len(filt))
    assert st == 0 and got == filt and r.checksum == zlib.adler32(filt)


def test_gzip_and_raw(lib):
    filt, _ = photo_stream(160, 100)
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    z = co.compress(filt) + co.flush()
    st, got, r = run(lib, z, len(filt), fmt=GZIP)
    assert st == 0 and got == filt and r.ck_done == 0 and r.declared == zlib.crc32(filt)
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    z = co.compress(filt) + co.flush()
    st, got, r = run(lib, z, len(filt), fmt=RAW)
    assert st == 0 and got == filt


def test_errors_fall_back_to_the_serial_decoder(lib):
    filt, z = photo_stream(256, 128)
    # truncated: need more input
    st, got, r = run(lib, z[: len(z) // 2], len(filt))
    ost, oout, ores = oracle.inflate(z[: len(z) // 2], oracle.ZLIB, len(filt))
    assert st == ost != 0 and r.stat[3] == 1
    # output too small
    st, got, r = run(lib, z, len(filt) // 3)
    ost, _, _ = oracle.inflate(z, oracle.ZLIB, len(filt) // 3)
    assert st == ost != 0
    # corrupted bits in the middle: whatever the oracle says (status and, when it succeeds, the bytes)
    bad = bytearray(z)
    for k in range(20):
        bad[len(z) // 2 + 37 * k] ^= 0x5A
    st, got, r = run(lib, bytes(bad), len(filt))
    ost, oout, ores = oracle.inflate(bytes(bad), oracle.ZLIB, len(filt))
    assert st == ost and (st != 0 or got == oout)
    # bad checksum
    bad = bytearray(z)
    bad[-1] ^= 1
    st, got, r = run(lib, bytes(bad), len(filt))
    assert st == oracle.inflate(bytes(bad), oracle.ZLIB, len(filt))[0] != 0 and got == filt


def test_tiny_and_empty(lib):
    for plain in (b"", b"a", b"abc" * 5, bytes(range(256)) * 3):
        z = zlib.compress(plain, 6)
        st, got, r = run(lib, z, len(plain) + 8)
        assert st == 0 and got == plain and r.checksum == zlib.adler32(plain)


# ---- more than one CTA per stream: block search + symbolic segments + window propagation + marker resolve ----
@pytest.fixture(scope="module", params=["cells"])
def seglib():
    """the segment pipeline, with inflate_cells_kernel decoding the segments (as run_segments does; the test ids name
    the engine)"""
    L = emu.load("emu_inflate_segments")
    L.emu_inflate_segmented.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    return L


def run_segmented(L, z: bytes, plain_len: int, nseg: int, fmt: int = ZLIB, plant: int = 0):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (plain_len + 64))()
    prod, used = C.c_uint64(), C.c_uint32()
    rc = L.emu_inflate_segmented(C.addressof(src), len(z), C.addressof(out), plain_len, fmt, nseg, plant,
                                 C.byref(prod), C.byref(used))
    return rc, bytes(out)[: prod.value], used.value


@pytest.mark.parametrize("nseg", [2, 5])
def test_segments_photo(seglib, nseg):
    filt, z = photo_stream(512, 300)
    rc, got, used = run_segmented(seglib, z, len(filt), nseg)
    assert rc == 0 and got == filt and used == nseg


def test_segments_markers_travel_through_long_copies(seglib):
    """flat graphics: almost every byte of a segment is a copy of a copy of ... the window in front of it"""
    img = corpus.make("graphic", 1400, 900, 2)
    filt, _ = corpus.zlib_png_stream(img, 4, 6)
    plain = filt[:300_000] * 5   # the same compression ratio everywhere: the segments' symbol buffers are sized by share
    co = zlib.compressobj(6, zlib.DEFLATED, 15, 9)
    z = b""
    for o in range(0, len(plain), 50_000):   # a block boundary every 50 000 bytes
        z += co.compress(plain[o:o + 50_000]) + co.flush(zlib.Z_SYNC_FLUSH)
    z += co.flush()
    rc, got, used = run_segmented(seglib, z, len(plain), 4)
    assert rc == 0 and got == plain and used >= 2


def test_segments_reference_stream_and_gzip(seglib):
    filt, _ = photo_stream(400, 300)
    z = oracle.deflate(filt, 9)        # few, growing blocks: not every split point finds a boundary
    rc, got, used = run_segmented(seglib, z, len(filt), 6)
    assert rc == 0 and got == filt and 1 <= used <= 6
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    z = co.compress(filt) + co.flush()
    rc, got, used = run_segmented(seglib, z, len(filt), 3, fmt=GZIP)
    assert rc == 0 and got == filt


def test_segments_false_split_point_is_rejected(seglib):
    """a split point that is not a block boundary (here: forged) must send the stream to the whole-stream path"""
    filt, z = photo_stream(512, 300)
    rc, _, _ = run_segmented(seglib, z, len(filt), 2, plant=8 * (len(z) // 3) + 3)
    assert rc == 1


def test_block_search_ignores_header_lookalike_in_stored_data(seglib):
    """a complete dynamic-block header copied into a stored block: the search may find it, the chain check must
    then reject the split (the decoder in front passes over it inside a stored block) -- or never see it"""
    filt, z = photo_stream(256, 128)
    inner = zlib.compress(filt, 6)[2:-4]              # raw deflate: starts with a real dynamic header
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    plain = filt + noise[:70_000] + inner + noise[70_000:] + filt
    z2 = zlib.compress(plain, 6)
    for nseg in (2, 3, 4):
        rc, got, _ = run_segmented(seglib, z2, len(plain), nseg)
        assert rc == 1 or got == plain


# ---- the round-1 engine (inflate_parallel_kernel: big batches) under the same emulator ----
def test_round1_engine_decodes_and_checksums(lib):
    L = emu.load("emu_inflate_old")
    L.emu_inflate_parallel.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(emu.Result), C.c_int]
    rng = np.random.default_rng(13)
    filt, _ = photo_stream(256, 96)
    cases = [photo_stream(320, 200)] + [corpus.zlib_png_stream(corpus.make("graphic", 640, 480, 1), 4, 6)]
    mixed = filt + rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes() + bytes(200_000) + filt
    cases.append((mixed, zlib.compress(mixed, 6)))
    for plain, z in cases:
        for order in (0, 4):
            src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
            out = (C.c_uint8 * (len(plain) + 64))()
            r = emu.Result()
            st = L.emu_inflate_parallel(C.addressof(src), len(z), C.addressof(out), len(plain), ZLIB, C.byref(r), order)
            assert st == 0 and bytes(out)[: r.produced] == plain
            assert r.ck_done == 1 and r.checksum == zlib.adler32(plain) and r.stat[3] == 0
    bad = bytearray(cases[0][1])
    bad[-2] ^= 4                                   # wrong Adler-32 in the trailer
    src = (C.c_uint8 * (len(bad) + 8)).from_buffer_copy(bytes(bad) + b"\0" * 8)
    out = (C.c_uint8 * (len(cases[0][0]) + 64))()
    r = emu.Result()
    st = L.emu_inflate_parallel(C.addressof(src), len(bad), C.addressof(out), len(cases[0][0]), ZLIB, C.byref(r), 0)
    assert st == oracle.inflate(bytes(bad), oracle.ZLIB, len(cases[0][0]))[0] != 0
