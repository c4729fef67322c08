"""The scanline kernels on the H100 at rows long enough to wrap 32-bit arithmetic (tests/wide_rows.py): filter selection
through filter_batch, encode_batch and png_encode_batch on 32 MiB rows whose None score sits at 2^32 and on a 1 GiB row
whose per-lane sums pass 2^32; Adam7 unfiltering through unfilter_batch and decode_batch where pass 7's pitch is 2^32
bits; the wavefront unfilter on one-row images with pitches around 2^31.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared).
Device buffers are torch tensors, compared on the device where a host copy would be GiBs; every test gives its
memory back before it returns."""
from __future__ import annotations

import ctypes as C
import zlib

import numpy as np
import pytest

import wide_rows
from oracle import oracle

pytestmark = pytest.mark.gpu
GiB = 1 << 30


@pytest.fixture
def budget(pngb200):
    """budget(gib) -> a context of its own, after skipping unless `gib` GiB of device memory are free; the context's
    arenas and torch's cached blocks go back to the driver when the test ends"""
    import torch
    made = []

    def take(gib: float):
        free, _ = torch.cuda.mem_get_info()
        if free < gib * GiB:
            pytest.skip(f"needs {gib} GiB of free device memory, {free / GiB:.1f} GiB free")
        made.append(pngb200.Context(0))
        return made[-1]

    yield take
    for c in made:
        c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def first_difference(got, want) -> int:
    """index of the first differing element of two equal-length device tensors, -1 when equal"""
    import torch
    ne = torch.nonzero(got != want)
    return int(ne[0, 0]) if ne.numel() else -1


def test_filter_batch_scores_past_2_32(pngb200, budget):
    """peak 0.5 GiB: the five 32 MiB rows of wide_rows.filter_cases in one batch, filter for filter as the reference"""
    ctx = budget(0.5)
    cases = wide_rows.filter_cases()
    images = [dict(pixels=row.tobytes(), width=len(row) // 4, height=1, volume=32, depth=8) for _, row, _ in cases]
    for (name, row, _), got in zip(cases, pngb200.filter_batch(ctx, images)):
        want = oracle.png_filter(row.tobytes(), len(row) // 4, 1, 32, 8)
        assert want[0] == 1
        assert got[0] == want[0], f"{name}: filter {got[0]}, the reference's {want[0]}"
        assert got == want, name


@pytest.mark.parametrize("name", ["none-up-tie-2^32", "wrapped-none-ties-sub"])
def test_encode_batch_and_png_encode_batch_past_2_32(pngb200, budget, name):
    """peak 1 GiB: the IDAT payload and the whole PNG file of a 32 MiB row whose None score wraps to 0 / ties Sub in
    32 bits equal the reference encoder's bytes"""
    ctx = budget(1)
    row = next(r for n, r, _ in wide_rows.filter_cases() if n == name)
    st, w = row.tobytes(), len(row) // 4
    ((es, idat),) = pngb200.encode_batch(ctx, [dict(pixels=st, width=w, height=1, volume=32, depth=8)], level=4)
    assert es == pngb200.OK
    assert idat == oracle.deflate(oracle.png_filter(st, w, 1, 32, 8), 4)
    ((ps, png),) = pngb200.png_encode_batch(ctx, [dict(storage=st, width=w, height=1, color=6, depth=8)], level=4)
    assert ps == pngb200.OK
    assert png == oracle.png_compress(st, w, 1, oracle.make_format(6, 8), False, 4)


def test_filter_lane_sums_past_2_32(pngb200, budget):
    """peak 2.5 GiB: one RGBA8 row of 2^30 + 4 bytes of 0x80.  Each of the warp's 32 lanes scores 2^25 bytes or more,
    2^32 or more for None, so the lanes' own sums wrap too, and None totals 2^37 + 512, which ties Sub's 512 in 32 bits.
    Sub wins: 1, four 0x80, then zeros"""
    import torch
    ctx = budget(2.5)
    pitch = 2 ** 30 + 4
    px = torch.full((pitch,), 0x80, dtype=torch.uint8, device="cuda")
    out = torch.full((pitch + 1 + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d = (pngb200.FilterDesc * 1)()
    d[0].pixels, d[0].pixels_len, d[0].filtered, d[0].filtered_cap = px.data_ptr(), pitch, out.data_ptr(), pitch + 1
    d[0].width, d[0].height, d[0].volume, d[0].depth = pitch // 4, 1, 32, 8
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_filter_batch(ctx.handle, d, 1, pngb200.MEM_DEVICE))
    assert out[:5].tolist() == [1, 0x80, 0x80, 0x80, 0x80]
    assert int(torch.count_nonzero(out[5:pitch + 1])) == 0
    assert bool((out[pitch + 1:] == 0xA5).all()), "written past the filtered row"
    del px, out


def unfilter_on_device(pngb200, ctx, filtered: bytes, w, h, vol, depth, il, pixels):
    import torch
    src = torch.frombuffer(bytearray(filtered), dtype=torch.uint8).cuda()
    d = (pngb200.ImageDesc * 1)()
    d[0].idat, d[0].idat_len, d[0].pixels, d[0].pixels_cap = src.data_ptr(), len(filtered), pixels.data_ptr(), pixels.numel()
    d[0].width, d[0].height, d[0].volume, d[0].depth, d[0].interlaced = w, h, vol, depth, int(il)
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_unfilter_batch(ctx.handle, d, 1, pngb200.MEM_DEVICE))
    torch.cuda.synchronize()
    assert d[0].status == pngb200.OK
    del src


def check_pass7_types(w, h, vol, types):
    """pass 7's first row must be reconstructed from its own bytes (Sub, Average, Paeth: None, and Up on a pass's first
    row, leave it as it is, which a wrapped pitch does too); a second pass-7 row must also read the row above"""
    rows = [types[k % len(types)] for k, z in enumerate(wide_rows.row_passes(w, h, vol)) if z == 6]
    assert rows[0] in (1, 3, 4), rows
    assert all(t in (2, 3, 4) for t in rows[1:]), rows


# all five filter types at height 2 (one row per pass), pass 7's row Sub, Average or Paeth
ADAM7_TYPES = {(2 ** 26 - 1, 64): (0, 1, 2, 4, 3), (2 ** 26, 64): (2, 0, 3, 4, 1), (2 ** 26 + 1, 64): (0, 2, 1, 3, 4),
               (2 ** 27, 32): (2, 0, 1, 4, 3)}


@pytest.mark.parametrize("w,vol", list(ADAM7_TYPES))
def test_unfilter_batch_adam7_pass7_pitch_2_32_bits(pngb200, budget, w, vol):
    """peak 4.5 GiB: two-row Adam7 images whose pass-7 scanline is 2^32 bits wide (RGBA16 at 2^26, RGBA8 at 2^27), with
    all five filter types, against the oracle on the device"""
    import torch
    ctx = budget(4.5)
    h, depth, types = 2, vol // 4, ADAM7_TYPES[w, vol]
    check_pass7_types(w, h, vol, types)
    filtered = wide_rows.filtered_stream(w, h, vol, True, types, w)
    st, want = oracle.png_unfilter(bytes(filtered), w, h, vol, depth, True)
    assert st == 0
    want = torch.frombuffer(bytearray(want), dtype=torch.uint8).cuda()
    pixels = torch.full((want.numel(),), 0xA5, dtype=torch.uint8, device="cuda")
    unfilter_on_device(pngb200, ctx, bytes(filtered), w, h, vol, depth, True, pixels)
    del filtered
    bad = first_difference(pixels, want)
    assert bad < 0, f"pixels differ from byte {bad} on"
    del want, pixels


def test_unfilter_batch_adam7_two_pass7_rows(pngb200, budget):
    """peak 4.5 GiB: a four-row Adam7 RGBA16 image of width 2^26 + 1 (2 GiB filtered, 2 GiB of pixels, staged through host
    memory).  Pass 7 has two rows, Sub then Paeth: the second is found pitch + 1 bytes after the first and reads it as
    the row above, so a wrapped pitch shows even where the first row alone would not"""
    ctx = budget(4.5)
    w, h, vol = 2 ** 26 + 1, 4, 64
    types = (0, 2, 3, 1, 4, 3, 1, 4)      # passes 1, 2, 4, 5, 6, 6, 7, 7
    assert wide_rows.row_passes(w, h, vol) == [0, 1, 3, 4, 5, 5, 6, 6]
    check_pass7_types(w, h, vol, types)
    filtered = bytes(wide_rows.filtered_stream(w, h, vol, True, types, 4))
    st, want = oracle.png_unfilter(filtered, w, h, vol, 16, True)
    assert st == 0
    ((us, got),) = pngb200.unfilter_batch(ctx, [dict(filtered=filtered, width=w, height=h, volume=vol, depth=16,
                                                     interlaced=1)])
    del filtered
    assert us == pngb200.OK
    if got != want:
        step = 1 << 24
        bad = next(i for i in range(0, len(want), step) if got[i:i + step] != want[i:i + step])
        bad += next(i for i in range(step) if got[bad + i] != want[bad + i])
        pytest.fail(f"pixels differ from byte {bad} on")


def test_decode_batch_adam7_pass7_pitch_2_32_bits(pngb200, budget):
    """peak 4 GiB: the 2^26-wide RGBA16 Adam7 image through the whole decode (a stored zlib stream of 1 GiB), pass 7's
    row Average"""
    ctx = budget(4)
    w, h, vol = 2 ** 26, 2, 64
    types = (4, 1, 2, 0, 3)
    check_pass7_types(w, h, vol, types)
    filtered = bytes(wide_rows.filtered_stream(w, h, vol, True, types, 7))
    idat = zlib.compress(filtered, 0)
    st, want = oracle.png_unfilter(filtered, w, h, vol, 16, True)
    del filtered
    assert st == 0
    (got,) = pngb200.decode_batch(ctx, [dict(idat=idat, width=w, height=h, volume=vol, depth=16, interlaced=1)])
    assert got.status == pngb200.OK
    assert got.pixels == want


CHUNK = 1 << 25


def wave_row(kind: str, lo: int, hi: int):
    """bytes [lo, hi) of (filtered row after its type byte, expected pixels) as int64 device tensors"""
    import torch
    k = torch.arange(lo, hi, dtype=torch.int64, device="cuda")
    if kind == "sub":          # deltas that make pixel byte k equal (k + 1) mod 256 at 8 bytes per pixel
        return torch.where(k < 8, k + 1, torch.full_like(k, 8)), (k + 1) & 0xFF
    pattern = (k ^ (k >> 8)) & 0xFF
    return pattern, pattern


@pytest.mark.parametrize("pitch,kind", [(2 ** 31 - 16, "none"), (2 ** 31, "up"), (2 ** 31 + 16, "sub")])
def test_unfilter_batch_wavefront_pitch_2_31(pngb200, budget, pitch, kind):
    """peak 5 GiB: a one-row RGBA16 image of `pitch` bytes through the wavefront kernel (None, Up -- the row above the
    first is zero -- and Sub); every byte and nothing past the row against the closed form, on the device.  One lane
    walks 2^27 chunks, about a minute each."""
    import torch
    ctx = budget(5)
    w = pitch // 8
    filtered = torch.empty(pitch + 1, dtype=torch.uint8, device="cuda")
    filtered[0] = {"none": 0, "sub": 1, "up": 2}[kind]
    for lo in range(0, pitch, CHUNK):
        hi = min(pitch, lo + CHUNK)
        filtered[1 + lo:1 + hi] = wave_row(kind, lo, hi)[0].to(torch.uint8)
    pixels = torch.full((pitch + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d = (pngb200.ImageDesc * 1)()
    d[0].idat, d[0].idat_len, d[0].pixels, d[0].pixels_cap = filtered.data_ptr(), pitch + 1, pixels.data_ptr(), pitch
    d[0].width, d[0].height, d[0].volume, d[0].depth = w, 1, 64, 16
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_unfilter_batch(ctx.handle, d, 1, pngb200.MEM_DEVICE))
    torch.cuda.synchronize()
    assert d[0].status == pngb200.OK
    del filtered
    for lo in range(0, pitch, CHUNK):
        hi = min(pitch, lo + CHUNK)
        bad = first_difference(pixels[lo:hi], wave_row(kind, lo, hi)[1].to(torch.uint8))
        assert bad < 0, f"pixel byte {lo + bad}: {int(pixels[lo + bad])}, expected {int(wave_row(kind, lo + bad, lo + bad + 1)[1])}"
    assert bool((pixels[pitch:] == 0xA5).all()), "written past the row"
    del pixels
