"""pngb200_png_inspect_files / pngb200_png_decode_files / pngb200_png_encode_files with the PNG files in device memory:
every result -- each descriptor field, each pixel byte, each error -- equals what the host-file calls give for the same
bytes, with pixels in host memory and in device memory, and the files at every offset 0..15 of one packed tensor."""
from __future__ import annotations

import ctypes as C
import os
import struct
import zlib

import numpy as np
import pytest

import container_cases as cc
import pngio
from conftest import GOLDEN, reference_outputs
from test_gpu_memspace import colour_formats, png_files, sample_top

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


def packed(files):
    """one CUDA uint8 tensor holding every file, file k starting at offset k % 16 of a 256-byte-aligned slot;
    returns (tensor, [(address, length)])"""
    at, spans = 0, []
    for k, f in enumerate(files):
        at = (at + 255) // 256 * 256 + k % 16
        spans.append((at, len(f)))
        at += len(f)
    host = np.zeros(max(at, 1), dtype=np.uint8)
    for (o, n), f in zip(spans, files):
        host[o: o + n] = np.frombuffer(f, dtype=np.uint8)
    t = torch.from_numpy(host).cuda()
    return t, [(t.data_ptr() + o, n) for o, n in spans]


def fields(im):
    return {k: v for k, v in vars(im).items() if k != "storage"}


def same_as_host(pngb200, ctx, files, device_pixels=False):
    """decodes `files` from device buffers and from host bytes; asserts equality; returns the host results"""
    want = pngb200.png_decode_batch(ctx, files)
    t, spans = packed(files)
    if not device_pixels:
        got = pngb200.png_decode_files(ctx, spans)
        for k, (g, w) in enumerate(zip(got, want)):
            assert fields(g) == fields(w), k
            assert g.storage == w.storage, k
    else:
        outs = [torch.full((max(w.width * w.height * 8, 1),), 0xA5, dtype=torch.uint8, device="cuda") for w in want]
        got = pngb200.png_decode_files(ctx, spans, [(o.data_ptr(), o.numel()) for o in outs])
        for k, (g, w, o) in enumerate(zip(got, want, outs)):
            assert fields(g) == fields(w), k
            if w.status == pngb200.OK:
                assert o[: len(w.storage)].cpu().numpy().tobytes() == w.storage, k
    inspected = pngb200.png_inspect_files(ctx, spans)
    for k, (g, h) in enumerate(zip(inspected, pngb200.png_inspect(files))):
        assert fields(g) == fields(h), k
    del t
    return want


def golden_files():
    out = []
    for sub in ("pngsuite", "ios", "invalid"):
        for f in sorted(os.listdir(os.path.join(GOLDEN, sub))):
            if f.endswith(".png"):
                out.append(open(os.path.join(GOLDEN, sub, f), "rb").read())
    out += [open(p, "rb").read() for p in reference_outputs().values()]
    return out


@pytest.mark.parametrize("device_pixels", [False, True])
def test_every_golden_file(pngb200, ctx, device_pixels):
    same_as_host(pngb200, ctx, golden_files(), device_pixels)


def five_idat_file():
    filtered = np.random.default_rng(3).integers(0, 4, (30, 1 + 30), dtype=np.uint8)
    filtered[:, 0] = 0
    z = zlib.compress(filtered.tobytes(), 9)
    step = (len(z) + 4) // 5
    parts = [z[i: i + step] for i in range(0, len(z), step)]
    assert len(parts) == 5
    ihdr = cc.chunk(b"IHDR", struct.pack(">IIBBBBB", 30, 30, 8, 0, 0, 0, 0))
    chunks = [ihdr, cc.chunk(b"gAMA", bytes(4))] + [cc.chunk(b"IDAT", p) for p in parts] + [cc.chunk(b"tEXt", b"k\0v"), cc.IEND]
    return chunks


def test_memspace_cases_and_each_chunk_crc_corrupted(pngb200, ctx, orc):
    """the memspace suite's files, and a five-IDAT file with each chunk's CRC spoiled in turn (IHDR, the chunk before
    the run, the first, middle and last IDAT, the chunk after the run, IEND): equal to the host path and the oracle"""
    chunks = five_idat_file()
    files = list(png_files())
    for k in range(len(chunks)):
        spoiled = list(chunks)
        c = bytearray(spoiled[k])
        c[-1] ^= 0x5A
        spoiled[k] = bytes(c)
        files.append(cc.png(spoiled))
    files.append(cc.png(chunks))
    for device_pixels in (False, True):
        want = same_as_host(pngb200, ctx, files, device_pixels)
    for f, w in zip(files[len(png_files()):], want[len(png_files()):]):
        info, storage = orc.png_decompress(f)
        assert (w.status, w.err_a, w.err_b) == (info.status, info.a, info.b)
        if info.status == 0:
            assert w.storage == storage
    assert sum(w.status == pngb200.ERR_LEX_INVALID_CHUNK_CHECKSUM for w in want[len(png_files()):]) == len(chunks)


def test_hundred_thousand_one_byte_idats_and_odd_files(pngb200, ctx):
    # 546 x 61 RGB, filter bytes 1: 99,979 filtered bytes in stored blocks, a zlib stream of exactly 100,000 bytes
    filtered = np.random.default_rng(5).integers(0, 256, (61, 1 + 3 * 546), dtype=np.uint8)
    filtered[:, 0] = 1
    z = zlib.compress(filtered.tobytes(), 0)
    assert len(z) == 100000
    many = pngio.write(546, 61, 8, 2, z, idat_chunk=1)
    ok = pngio.write(546, 61, 8, 2, z, idat_chunk=7777)
    files = [many, b"", ok, b"\x89PNG", ok[:-5], golden_files()[3], ok[:60] + b"\xff" + ok[61:]]
    want = same_as_host(pngb200, ctx, files)
    assert want[0].status == pngb200.OK and want[0].idat_chunks == 100000 and want[0].storage == want[2].storage
    # a null pointer with zero length is an empty file
    got = pngb200.png_decode_files(ctx, [(0, 0)])
    assert fields(got[0]) == fields(want[1])


def test_8k_rgba_with_8_kib_idats(pngb200, ctx):
    rng = np.random.default_rng(8)
    w, h = 7680, 4320
    x = np.arange(w, dtype=np.uint32)[None, :, None]
    y = np.arange(h, dtype=np.uint32)[:, None, None]
    img = ((x * 3 + y * 5 + np.arange(4, dtype=np.uint32)) & 0xFF).astype(np.uint8)
    img ^= rng.integers(0, 8, (h, 1, 4), dtype=np.uint8)
    filtered = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, w * 4)], axis=1)
    z = zlib.compress(filtered.tobytes(), 1)
    f = pngio.write(w, h, 8, 6, z, idat_chunk=8192)
    want = same_as_host(pngb200, ctx, [f], device_pixels=True)
    assert want[0].status == pngb200.OK and want[0].idat_chunks == (len(z) + 8191) // 8192


def test_capacity_and_bad_file_memspace(pngb200, ctx):
    f = png_files()[0]
    t, spans = packed([f])
    probe = pngb200.png_inspect([f])[0]
    size = pngb200.storage_size(probe.width, probe.height, probe.depth * pngb200._CHANNELS[probe.color])
    out = torch.empty(size, dtype=torch.uint8, device="cuda")
    host_file = C.create_string_buffer(f, len(f))
    for memspace in (pngb200.MEM_HOST, pngb200.MEM_DEVICE):
        rcs = []
        for file_memspace, addr in ((pngb200.MEM_HOST, C.addressof(host_file)), (pngb200.MEM_DEVICE, spans[0][0])):
            d = (pngb200.PngDesc * 1)()
            d[0].file, d[0].file_len = addr, len(f)
            d[0].pixels, d[0].pixels_cap = out.data_ptr(), size - 1
            rcs.append(ctx._lib.pngb200_png_decode_files(ctx.handle, d, 1, file_memspace, memspace))
        assert rcs == [pngb200.ERR_OUTPUT_CAPACITY] * 2
    d = (pngb200.PngDesc * 1)()
    d[0].file, d[0].file_len = spans[0]
    assert ctx._lib.pngb200_png_decode_files(ctx.handle, d, 1, 2, pngb200.MEM_HOST) == pngb200.ERR_BAD_ARGUMENT
    assert ctx._lib.pngb200_png_inspect_files(ctx.handle, d, 1, 7) == pngb200.ERR_BAD_ARGUMENT
    e = (pngb200.PngEncodeDesc * 1)()
    assert ctx._lib.pngb200_png_encode_files(ctx.handle, e, 1, pngb200.MEM_HOST, -1) == pngb200.ERR_BAD_ARGUMENT
    del t


@pytest.mark.parametrize("idat_chunk", [0, 1000, 16])
def test_encode_into_device_files(pngb200, ctx, idat_chunk):
    """bytes equal to png_encode_batch for every colour format, interlaced and not; the files decode back through
    png_decode_files to the input storage without leaving the GPU"""
    rng = np.random.default_rng(40 + idat_chunk)
    images = []
    for k, (color, depth, bgr, key, pal) in enumerate(colour_formats()):
        for il in (False, True):
            w, h = 23 + 11 * k, 9 + 2 * k
            n = pngb200.storage_size(w, h, depth * pngb200._CHANNELS[color])
            st = rng.integers(0, sample_top(color, depth), n, dtype=np.uint8).tobytes()
            images.append(dict(storage=st, width=w, height=h, color=color, depth=depth, bgr=bgr, key=key, palette=pal,
                               interlaced=il))
    want = pngb200.png_encode_batch(ctx, images, level=6, idat_chunk=idat_chunk)
    caps = [pngb200.png_encode_bound(g, idat_chunk) for g in images]
    bufs = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    got = pngb200.png_encode_files(ctx, images, [(b.data_ptr(), c) for b, c in zip(bufs, caps)], level=6, idat_chunk=idat_chunk)
    for (st, n), (wst, wfile), b in zip(got, want, bufs):
        assert st == wst == pngb200.OK and n == len(wfile)
        assert b[:n].cpu().numpy().tobytes() == wfile
    outs = [torch.empty(max(len(g["storage"]), 1), dtype=torch.uint8, device="cuda") for g in images]
    back = pngb200.png_decode_files(ctx, [(b.data_ptr(), n) for b, (_, n) in zip(bufs, got)],
                                    [(o.data_ptr(), o.numel()) for o in outs])
    for g, im, o in zip(images, back, outs):
        assert im.status == pngb200.OK
        assert torch.equal(o, torch.frombuffer(bytearray(g["storage"]), dtype=torch.uint8).cuda())


def test_trim_then_same_device_batch(pngb200):
    ctx = pngb200.Context(0)
    try:
        files = png_files() + golden_files()[:20]
        t, spans = packed(files)
        first = [(fields(im), im.storage) for im in pngb200.png_decode_files(ctx, spans)]
        ctx.trim()
        assert [(fields(im), im.storage) for im in pngb200.png_decode_files(ctx, spans)] == first
        del t
    finally:
        ctx.close()
