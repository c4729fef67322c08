"""The unfilter stage's pass path on the H100: Adam7 and 1/2/4-bit images whose filtered stream is longer than 64 KiB are
reconstructed pass by pass on the wavefront (unfilter_pass_kernel), in place, and interleaved into PNG.Image.storage
(unfilter_interleave_kernel).  Outputs are compared with the oracle through decode_batch, unfilter_batch with host and
device memory, and png_decode_files; Context.unfilter_stats shows which path each image took.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import ctypes as C
import struct
import zlib

import numpy as np
import pytest

import wide_rows
from oracle import oracle

pytestmark = pytest.mark.gpu
GiB = 1 << 30
GENERIC_MAX = 65536   # filtered bytes up to which Adam7 and 1/2/4-bit images stay on the generic kernel (pngb200.h)
TYPES = (1, 4, 2, 3, 0, 4, 4, 3, 1, 2, 9)   # 9: an invalid filter byte
# (volume, depth): RGBA8, RGB16, VA16, V8 (indexed 8-bit alike), indexed or grey 4, 2 and 1-bit
FORMATS = [(32, 8), (48, 16), (32, 16), (8, 8), (4, 4), (2, 2), (1, 1)]


@pytest.fixture
def budget(pngb200):
    """budget(gib) -> a context of its own, after skipping unless `gib` GiB of device memory are free"""
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


def job(w, h, volume, depth, interlaced, seed, cut=0, types=TYPES, level=1):
    """a decode_batch job over seeded scanlines; the zlib stream holds the filtered bytes without the last `cut`"""
    f = bytes(wide_rows.filtered_stream(w, h, volume, interlaced, types, seed))
    f = f[:len(f) - cut]
    return dict(idat=zlib.compress(f, level), width=w, height=h, volume=volume, depth=depth, interlaced=int(interlaced),
                fmt=0, filtered=f)


def check_decoded(jobs, got):
    for j, g in zip(jobs, got):
        st, want, _ = oracle.png_decode(j["idat"], j["width"], j["height"], j["volume"], j["depth"], bool(j["interlaced"]))
        key = (j["width"], j["height"], j["volume"], j["interlaced"])
        assert g.status == st, key
        assert g.pixels == want, key


@pytest.mark.parametrize("w,h,gib", [(1920, 1080, 1), (7680, 4320, 5)])
def test_decode_batch_every_format(pngb200, budget, w, h, gib):
    """peak 1 GiB (1080p) / 5 GiB (8K): Adam7 RGBA8, RGB16, VA16, V8 and 4/2/1-bit in one batch, with the 8K batch
    also holding non-interlaced 1/2/4-bit images: every image on the pass path, pixels as the oracle's"""
    ctx = budget(gib)
    jobs = [job(w, h, v, d, True, v + d) for v, d in FORMATS]
    if w == 7680:
        jobs += [job(w, h, d, d, False, 50 + d) for d in (1, 2, 4)]
    got = pngb200.decode_batch(ctx, jobs)
    assert ctx.unfilter_stats() == dict(wavefront=0, passes=len(jobs), generic=0)
    check_decoded(jobs, got)


def test_unfilter_batch_host_and_device(pngb200, budget):
    """peak 1 GiB: unfilter_batch over a 1080p Adam7 RGBA8 and a 1080p non-interlaced 2-bit stream, from host memory and
    from device memory; the pass path reconstructs in a private copy, so the caller's device stream is unchanged"""
    import torch
    ctx = budget(1)
    images = [(1920, 1080, 32, 8, True), (1920, 1080, 2, 2, False)]
    streams = [bytes(wide_rows.filtered_stream(w, h, v, il, TYPES, k)) for k, (w, h, v, _, il) in enumerate(images)]
    wants = [oracle.png_unfilter(f, w, h, v, d, il)[1] for f, (w, h, v, d, il) in zip(streams, images)]
    got = pngb200.unfilter_batch(ctx, [dict(filtered=f, width=w, height=h, volume=v, depth=d, interlaced=int(il))
                                       for f, (w, h, v, d, il) in zip(streams, images)])
    assert ctx.unfilter_stats() == dict(wavefront=0, passes=2, generic=0)
    assert [g for _, g in got] == wants
    assert [s for s, _ in got] == [pngb200.OK] * 2

    srcs = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in streams]
    before = [s.clone() for s in srcs]
    outs = [torch.full((len(wnt) + 64,), 0xA5, dtype=torch.uint8, device="cuda") for wnt in wants]
    d = (pngb200.ImageDesc * 2)()
    for k, ((w, h, v, dep, il), s, o) in enumerate(zip(images, srcs, outs)):
        d[k].idat, d[k].idat_len, d[k].pixels, d[k].pixels_cap = s.data_ptr(), s.numel(), o.data_ptr(), len(wants[k])
        d[k].width, d[k].height, d[k].volume, d[k].depth, d[k].interlaced = w, h, v, dep, int(il)
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_unfilter_batch(ctx.handle, d, 2, pngb200.MEM_DEVICE))
    torch.cuda.synchronize()
    assert ctx.unfilter_stats() == dict(wavefront=0, passes=2, generic=0)
    for k in range(2):
        assert d[k].status == pngb200.OK
        assert torch.equal(srcs[k], before[k]), "the caller's filtered stream was written"
        assert outs[k][:len(wants[k])].cpu().numpy().tobytes() == wants[k], k
        assert bool((outs[k][len(wants[k]):] == 0xA5).all()), "written past the pixels"


def png_file(w, h, color, depth, interlaced, idat: bytes) -> bytes:
    def chunk(kind, body):
        return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))
    ihdr = struct.pack(">IIBBBBB", w, h, depth, color, 0, 0, int(interlaced))
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IDAT", idat) + chunk(b"IEND", b"")


def test_png_decode_files_interlaced_8k_in_device_memory(pngb200, budget):
    """peak 2 GiB: one interlaced 8K RGBA8 PNG file in device memory decodes to the oracle's storage"""
    import torch
    ctx = budget(2)
    w, h = 7680, 4320
    f = bytes(wide_rows.filtered_stream(w, h, 32, True, TYPES, 8))
    st, want = oracle.png_unfilter(f, w, h, 32, 8, True)
    assert st == 0
    data = png_file(w, h, 6, 8, True, zlib.compress(f, 1))
    del f
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    (got,) = pngb200.png_decode_files(ctx, [(t.data_ptr(), t.numel())])
    assert got.status == pngb200.OK
    assert ctx.unfilter_stats() == dict(wavefront=0, passes=1, generic=0)
    assert got.storage == want


def test_mixed_batch_keeps_the_filter_histogram(pngb200, budget):
    """peak 1 GiB: interlaced, sub-byte and non-interlaced RGBA8 images in one batch, on all three paths; the filter
    histogram counts the non-interlaced RGBA8 images' rows only"""
    ctx = budget(1)
    rng = np.random.default_rng(5)
    jobs, hist = [], np.zeros(6, dtype=np.int64)
    for k in range(3):
        w, h = 300 + 17 * k, 200 + 31 * k
        types = tuple(int(t) for t in rng.integers(0, 6, size=h))
        jobs.append(job(w, h, 32, 8, False, 70 + k, types=types))
        for t in types:
            hist[min(t, 5)] += 1
    jobs += [job(640, 480, 32, 8, True, 1), job(2000, 1500, 1, 1, False, 2), job(20, 20, 48, 16, True, 3),
             job(33, 9, 4, 4, False, 4)]
    got = pngb200.decode_batch(ctx, jobs)
    assert ctx.unfilter_stats() == dict(wavefront=3, passes=2, generic=2)
    assert ctx.filter_histogram() == [int(x) for x in hist]
    check_decoded(jobs, got)


def test_truncated_streams_and_an_inflate_error(pngb200, budget):
    """peak 1 GiB: 1080p Adam7 RGBA8 streams that end inside pass 1, pass 4 and pass 7, and one with a corrupt deflate
    block: rows up to the first incomplete one are reconstructed, after an error none, the rest are zero"""
    ctx = budget(1)
    w, h = 1920, 1080
    full = oracle.filtered_size(w, h, 32, True)
    ends = [0]
    for _, _, sh, pitch in wide_rows.adam7_passes(w, h, 32):
        ends.append(ends[-1] + sh * (pitch + 1))
    jobs = [job(w, h, 32, 8, True, z, cut=full - (ends[z] + (ends[z + 1] - ends[z]) // 2 + 5)) for z in (0, 3, 6)]
    bad = job(w, h, 32, 8, True, 9)
    idat = bytearray(bad["idat"])
    idat[2] |= 0x06     # BTYPE 11: a reserved block type
    bad["idat"] = bytes(idat)
    jobs.append(bad)
    got = pngb200.decode_batch(ctx, jobs)
    assert ctx.unfilter_stats() == dict(wavefront=0, passes=4, generic=0)
    check_decoded(jobs, got)
    assert got[3].status == pngb200.ERR_BLOCK_TYPE
    assert not any(got[3].pixels)


def test_threshold_sides(pngb200, budget):
    """peak 0.1 GiB: a stream of exactly 64 KiB stays on the generic kernel, one more row takes the pass path, for a
    non-interlaced 1-bit image (rows of 127 + 1 bytes) and for Adam7 RGBA8 images around the same size"""
    ctx = budget(0.1)
    at, over = job(1016, 512, 1, 1, False, 1), job(1016, 513, 1, 1, False, 2)
    assert len(at["filtered"]) == GENERIC_MAX and len(over["filtered"]) > GENERIC_MAX
    sizes = [(wh, oracle.filtered_size(wh, wh, 32, True)) for wh in range(122, 132)]
    small = [job(wh, wh, 32, 8, True, wh) for wh, n in sizes if n <= GENERIC_MAX]
    large = [job(wh, wh, 32, 8, True, wh) for wh, n in sizes if n > GENERIC_MAX]
    assert small and large
    for jobs, want in (([at] + small, dict(wavefront=0, passes=0, generic=1 + len(small))),
                       (([over] + large), dict(wavefront=0, passes=1 + len(large), generic=0))):
        got = pngb200.decode_batch(ctx, jobs)
        assert ctx.unfilter_stats() == want
        check_decoded(jobs, got)
