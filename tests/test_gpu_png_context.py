"""Online decoding on the H100 (pngb200_png_context: PNG.Context.push(data:overdraw:)): after every push the status,
the storage and the progress are the oracle's (oracle/png_context.c), for every golden pushed by its own IDAT chunks and
then 1 and 7 bytes at a time, for host and device storage, and for 1080p and 8K files pushed as the reference's 65 544-byte
IDAT chunks; the errors of PNG.Decoder.push and PNG.Context at IEND; and the launches a push costs.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import zlib

import numpy as np
import pytest

import pngio
from oracle import oracle
from png_context_cases import GOLDEN, OracleContext, geometry, goldens, random_storage, stored_prefix, stored_zlib

pytestmark = pytest.mark.gpu
GiB = 1 << 30
GOLDENS = goldens()
BYTEWISE = {"pngsuite/z00n2c08.png", "pngsuite/oi9n0g16.png", "pngsuite/oi9n2c16.png", "pngsuite/basi0g01.png",
            "pngsuite/basi4a16.png", "ios/basi6a08.png"}


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


def status(fn, *args):
    from importlib import import_module
    try:
        fn(*args)
        return 0
    except import_module("swift-png_b200").PNGB200Error as e:
        return e.status


def new_pair(pngb200, ctx, g, pixels=None):
    gpu = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"], pixels)
    return gpu, OracleContext(**g)


def storage_of(c, size, device_buf=None, at=0):
    if device_buf is None:
        return c.storage()
    return bytes(device_buf.cpu().numpy().tobytes()[at:at + size])


def push_and_compare(pngb200, ctx, g, pieces, overdraw, device=False, every=1):
    """push `pieces` into a GPU context and the oracle's, comparing status and progress after every push and storage
    after every `every`-th push and the last one"""
    buf = None
    size = oracle.storage_size(g["w"], g["h"], g["volume"])
    if device:
        import torch
        buf = torch.full((size + 1,), 0x5A, dtype=torch.uint8, device="cuda")   # storage at buf[1:]: an odd address
        gpu, ref = new_pair(pngb200, ctx, g, (buf.data_ptr() + 1, size))
    else:
        gpu, ref = new_pair(pngb200, ctx, g)
    try:
        for i, p in enumerate(pieces):
            od = overdraw if isinstance(overdraw, bool) else overdraw[i % len(overdraw)]
            want = ref.push(p, od)
            assert status(gpu.push, p, od) == want, i
            assert gpu.progress() == ref.progress(), i
            if i % every == 0 or i == len(pieces) - 1:
                assert storage_of(gpu, size, buf, 1) == ref.storage(), i
        assert status(gpu.end) == ref.end()
    finally:
        gpu.close()
        ref.close()


@pytest.mark.parametrize("name,data", GOLDENS, ids=[n for n, _ in GOLDENS])
def test_goldens(pngb200, budget, name, data):
    """peak 0.1 GiB: each golden pushed by its own IDAT chunks with overdraw, then 7 bytes at a time (4 099 for the
    colour goldens of 100-600 KB, whose oracle inflates every pushed prefix again) without and with alternating
    overdraw, and a few byte by byte (oi9n* have one-byte IDAT chunks; z00n2c08 is all stored blocks)"""
    ctx = budget(0.1)
    png = pngio.parse(data)
    g = geometry(png)
    push_and_compare(pngb200, ctx, g, pngio.idat_chunks(data), True)
    step = 7 if len(png.idat) <= 16384 else 4099
    sevens = [png.idat[i:i + step] for i in range(0, len(png.idat), step)]
    push_and_compare(pngb200, ctx, g, sevens, False)
    push_and_compare(pngb200, ctx, g, sevens, [True, False, True])
    if name in BYTEWISE or name.startswith("pngsuite/oi9n"):
        push_and_compare(pngb200, ctx, g, [png.idat[i:i + 1] for i in range(len(png.idat))], True)


def test_device_storage(pngb200, budget):
    """peak 0.1 GiB: storage in device memory, at an odd address, for Adam7 goldens of every depth"""
    ctx = budget(0.1)
    for name in ("basi0g01", "basi0g02", "basi0g04", "basi2c08", "basi4a16", "basi6a16", "basi3p08"):
        data = open(f"{GOLDEN}/pngsuite/{name}.png", "rb").read()
        png = pngio.parse(data)
        pieces = [png.idat[i:i + 11] for i in range(0, len(png.idat), 11)]
        push_and_compare(pngb200, ctx, geometry(png), pieces, True, device=True)


def big_file(w, h, interlaced):
    """a smooth RGBA8 image with a little noise, filtered by the oracle's encoder and compressed by zlib at level 1 (fast
    to make at 8K), framed in 65 544-byte IDAT chunks"""
    rng = np.random.default_rng(w + interlaced)
    y, x = np.mgrid[0:h, 0:w].astype(np.uint32)
    img = np.stack([(x // 3 + y // 5), (x * y) >> 11, (x + 2 * y) >> 4, 255 - (y >> 5)], axis=-1).astype(np.uint8)
    img += rng.integers(0, 3, img.shape, dtype=np.uint8)
    img = img.tobytes()
    idat = zlib.compress(oracle.png_filter(img, w, h, 32, 8, interlaced), 1)
    return img, pngio.write(w, h, 8, 6, idat, interlaced=interlaced, idat_chunk=65544)


CASES = [(1920, 1080, 1, il, mem) for il in (False, True) for mem in ("host", "device")] + \
        [(7680, 4320, 4, il, "host") for il in (False, True)]


@pytest.mark.parametrize("w,h,gib,interlaced,memspace", CASES)
def test_large_files(pngb200, budget, w, h, gib, interlaced, memspace):
    """peak 1 GiB (1080p) / 4 GiB (8K): an RGBA8 file pushed as its 65 544-byte IDAT chunks, overdraw off and on: the
    decoder's position at a sample of pushes and storage there and at the end, where it equals png_decode_batch's; every push
    costs the inflator's launches, one unfilter and at most seven assign launches (at 1080p counted exactly against a
    bare inflator pushed the same chunks)"""
    ctx = budget(gib)
    img, f = big_file(w, h, interlaced)
    chunks = pngio.idat_chunks(f)
    (dec,) = pngb200.png_decode_batch(ctx, [f])
    assert dec.status == 0 and dec.storage == img
    g = dict(w=w, h=h, volume=32, depth=8, interlaced=interlaced, standard=0)
    sample = set(np.linspace(0, len(chunks) - 1, 6 if w < 4000 else 4).astype(int).tolist())
    for overdraw in (False, True):
        buf = None
        size = w * h * 4
        if memspace == "device":
            import torch
            buf = torch.empty(size, dtype=torch.uint8, device="cuda")
            gpu = pngb200.PngContext(ctx, w, h, 32, 8, interlaced, 0, (buf.data_ptr(), size))
        else:
            gpu = pngb200.PngContext(ctx, w, h, 32, 8, interlaced)
        ref = OracleContext(**g)
        twin = pngb200.Inflator(ctx) if w < 4000 else None   # the launches the context's own inflator makes
        pending = b""
        try:
            for i, p in enumerate(chunks):
                before = ctx.launches
                if twin is not None:
                    twin.push(p)
                inflator = ctx.launches - before
                gpu.push(p, overdraw)
                prog = gpu.progress()
                own = ctx.launches - before - 2 * inflator if twin is not None else ctx.launches - before - 4
                assert own <= 1 + 7, (i, ctx.launches - before, inflator)
                pending += p
                if i in sample:   # the oracle's state depends on the prefix only: push what arrived since the last sample
                    assert ref.push(pending, overdraw) == 0
                    pending = b""
                    # (the rows the oracle's last push wrote span several chunks; the band is pinned by test_goldens)
                    assert prog[:4] == ref.progress()[:4] and (prog[4:] == (0, 0) or prog[4] < prog[5] <= h), (i, prog)
                    assert storage_of(gpu, size, buf) == ref.storage(), i
            gpu.end()
            assert storage_of(gpu, size, buf) == img
        finally:
            gpu.close()
            ref.close()
            if twin is not None:
                twin.close()
            del buf


def test_errors(pngb200, budget):
    """peak 0.1 GiB: -49 after the trailer (even for an empty push); -48 in the completing push and in a later one that
    brings filtered bytes; a corrupted byte mid-stream gives the oracle's status and payload, leaves the storage as the
    previous push did, and sticks; end() before the trailer is -50, after it OK"""
    ctx = budget(0.1)
    w, h = 53, 29
    final = random_storage(w, h, 32, 8, 4)
    filtered = oracle.png_filter(final, w, h, 32, 8, True)
    idat = zlib.compress(filtered, 9)
    g = dict(w=w, h=h, volume=32, depth=8, interlaced=True, standard=0)
    gpu = pngb200.PngContext(ctx, w, h, 32, 8, True)
    gpu.push(idat[:-2])
    assert status(gpu.end) == pngb200.ERR_PNG_INCOMPLETE_DATASTREAM and gpu.storage() == final
    gpu.push(idat[-2:])
    gpu.end()
    assert status(gpu.push, b"") == pngb200.ERR_PNG_EXTRANEOUS_COMPRESSED_DATA
    assert status(gpu.push, b"abc") == pngb200.ERR_PNG_EXTRANEOUS_COMPRESSED_DATA
    gpu.close()
    # extraneous image data
    extra = stored_zlib(filtered + bytes(300), 100)
    cut = stored_prefix((len(filtered) + 100) // 100 * 100, 100)
    push_and_compare(pngb200, ctx, g, [extra[:cut], extra[cut:cut + 1], extra[cut + 1:cut + 9], extra[cut + 9:]], True)
    gpu = pngb200.PngContext(ctx, w, h, 32, 8, True)
    assert status(gpu.push, extra[:cut]) == pngb200.ERR_PNG_EXTRANEOUS_IMAGE_DATA and gpu.storage() == final
    gpu.close()
    # a corrupted byte mid-stream
    bad = bytearray(idat)
    bad[len(bad) // 2] ^= 0x21
    gpu, ref = new_pair(pngb200, ctx, g)
    st = 0
    for at in range(0, len(bad), 64):
        before = gpu.storage()
        want = ref.push(bytes(bad[at:at + 64]), True)
        try:
            gpu.push(bytes(bad[at:at + 64]), True)
            st = 0
        except pngb200.PNGB200Error as e:
            st = e.status
            assert e.payload == ref.error()[1:]
        assert st == want and gpu.storage() == ref.storage()
        if st < 0:
            assert gpu.storage() == before
            break
    assert st < 0 and st == oracle.inflate(bytes(bad), oracle.ZLIB)[0]
    assert status(gpu.push, b"\x00") == st
    gpu.close()
    ref.close()


def test_create_rejects_bad_arguments(pngb200, budget):
    """peak 0.1 GiB: bad geometry, bad pixel formats and too small a storage return NULL with a reason"""
    ctx = budget(0.1)
    for args in ((0, 4, 32, 8), (4, 0, 32, 8), (4, 4, 12, 8), (4, 4, 3, 1), (4, 4, 32, 3)):
        with pytest.raises(pngb200.PNGB200Error):
            pngb200.PngContext(ctx, *args)
    import torch
    buf = torch.empty(63, dtype=torch.uint8, device="cuda")
    with pytest.raises(pngb200.PNGB200Error):
        pngb200.PngContext(ctx, 4, 4, 32, 8, False, 0, (buf.data_ptr(), 63))
