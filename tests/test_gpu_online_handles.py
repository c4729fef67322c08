"""The online handles on the H100 across pngb200_ctx_trim: an inflator, a PngContext (host and device storage) and an
online Deflator are pushed seeded streams in pieces with ctx.trim() before every push, and batch pushes of all three kinds
are made with a trim before every call.  The trim gives the ctx's push workspaces back (staging, tables, checksum
partials, the pinned buffers behind them); the handles own their buffers, so every push must leave what the same push
leaves on twin handles of a ctx that is never trimmed: statuses, error payloads, pulled bytes, progress, storage, popped
blocks and stats().

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import random
import zlib

import numpy as np
import pytest

import pngio
from png_context_cases import GOLDEN, geometry
from test_gpu_deflator_online import take, text
from test_gpu_inflate_resume import FORMATS
from test_gpu_png_context import big_file

pytestmark = pytest.mark.gpu
GiB = 1 << 30


@pytest.fixture
def budget(pngb200):
    """budget(gib) -> two contexts of their own (trimmed, never trimmed), after skipping unless `gib` GiB of device
    memory are free"""
    import torch
    made = []

    def take_(gib: float):
        free, _ = torch.cuda.mem_get_info()
        if free < gib * GiB:
            pytest.skip(f"needs {gib} GiB of free device memory, {free / GiB:.1f} GiB free")
        made.extend([pngb200.Context(0), pngb200.Context(0)])
        return made[-2], made[-1]

    yield take_
    for c in made:
        c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def status(pngb200, fn, *args):
    try:
        return fn(*args) or 0
    except pngb200.PNGB200Error as e:
        return e.status


def cut(data, rng, sizes):
    out, at = [], 0
    while at < len(data):
        n = rng.choice(sizes)
        out.append(data[at:at + n])
        at += n
    return out + [b""]


def inflate_streams():
    """(format, stream): stored blocks in every format, fixed and dynamic blocks, an output that outgrows its buffer
    inside a push, and a corrupt stream"""
    rng = np.random.default_rng(23)
    plain = rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    low = rng.integers(0, 8, 300_000, dtype=np.uint8).tobytes()
    out = []
    for fmt, wb in FORMATS.values():
        c = zlib.compressobj(0, zlib.DEFLATED, wb)
        out.append((fmt, c.compress(plain) + c.flush()))
    out.append((0, zlib.compress(low, 1)))
    out.append((0, zlib.compress(low, 9)))
    out.append((0, zlib.compress(bytes(2_000_000), 9)))
    bad = bytearray(zlib.compress(low, 6))
    bad[len(bad) // 2] ^= 0x5A
    out.append((0, bytes(bad)))
    return out


def inflator_state(z):
    return z.error(), z.stats(), z.ctx._lib.pngb200_inflator_available(z.handle)


def test_inflator_across_trims(pngb200, budget):
    """peak 0.2 GiB: pieces of 1 byte to 70 KB, across stored block headers and 64 KiB ring-kernel pushes"""
    trimmed, plain = budget(0.2)
    rng = random.Random(5)
    for fmt, s in inflate_streams():
        a, b = pngb200.Inflator(trimmed, fmt), pngb200.Inflator(plain, fmt)
        try:
            for i, p in enumerate(cut(s, rng, [1, 7, 1000, 20_000, 70_000])):
                trimmed.trim()
                assert status(pngb200, a.push, p) == status(pngb200, b.push, p), (fmt, i)
                assert inflator_state(a) == inflator_state(b), (fmt, i)
                if rng.random() < 0.3:
                    k = rng.randrange(0, b.ctx._lib.pngb200_inflator_available(b.handle) + 1)
                    assert a.pull(k) == b.pull(k), (fmt, i)
            assert a.pull_all() == b.pull_all()
        finally:
            a.close()
            b.close()


def context_files():
    """(geometry, idat, piece sizes): 640x360 RGBA8 plain and Adam7, z00n2c08 (all stored blocks) and a corrupt file"""
    out = []
    for il in (False, True):
        png = pngio.parse(big_file(640, 360, il)[1])
        out.append((geometry(png), png.idat, [1, 7, 1000, 20_000, 70_000]))
    png = pngio.parse(open(f"{GOLDEN}/pngsuite/z00n2c08.png", "rb").read())
    out.append((geometry(png), png.idat, [1, 7, 300]))
    bad = bytearray(out[0][1])
    bad[len(bad) // 3] ^= 0x5A
    out.append((out[0][0], bytes(bad), [20_000, 70_000]))
    return out


class Twin:
    """a PngContext, in host storage or in device storage at an odd address"""

    def __init__(self, pngb200, ctx, g, device):
        self.size, self.buf = None, None
        pixels = None
        if device:
            import torch
            self.size = pngb200.storage_size(g["w"], g["h"], g["volume"])
            self.buf = torch.full((self.size + 1,), 0x5A, dtype=torch.uint8, device="cuda")
            pixels = (self.buf.data_ptr() + 1, self.size)
        self.c = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"], pixels)

    def state(self):
        storage = self.c.storage() if self.buf is None else bytes(self.buf.cpu().numpy().tobytes()[1:])
        return self.c.error(), self.c.progress(), storage


def test_png_context_across_trims(pngb200, budget):
    """peak 0.2 GiB: host and device storage, with and without overdraw"""
    trimmed, plain = budget(0.2)
    rng = random.Random(6)
    for device in (False, True):
        for g, idat, sizes in context_files():
            a, b = Twin(pngb200, trimmed, g, device), Twin(pngb200, plain, g, device)
            try:
                for i, p in enumerate(cut(idat, rng, sizes)):
                    od = rng.random() < 0.5
                    trimmed.trim()
                    assert status(pngb200, a.c.push, p, od) == status(pngb200, b.c.push, p, od), (device, i)
                    assert a.state() == b.state(), (device, i)
                assert status(pngb200, a.c.end) == status(pngb200, b.c.end)
            finally:
                a.c.close()
                b.c.close()


def test_deflator_across_trims(pngb200, budget):
    """peak 0.5 GiB: full mode (level 9), lazy (4) and stored (0) levels in every format; the blocks popped and pulled
    after every push and stats(), device bytes held included"""
    trimmed, plain = budget(0.5)
    rng = random.Random(7)
    for fmt, level, exponent in ((pngb200.FORMAT_ZLIB, 9, 15), (pngb200.FORMAT_GZIP, 4, 8), (pngb200.FORMAT_IOS, 0, 15)):
        data = text(300_000, level)
        a = pngb200.Deflator(trimmed, fmt, level, exponent, chunk_bytes=4000, online=True)
        b = pngb200.Deflator(plain, fmt, level, exponent, chunk_bytes=4000, online=True)
        try:
            pieces = cut(data, rng, [1, 700, 4097, 30_000, 70_001])
            for i, p in enumerate(pieces):
                last = i == len(pieces) - 1
                trimmed.trim()
                a.push(p, last=last)
                b.push(p, last=last)
                assert take(a, last) == take(b, last), (level, i)
                assert a.stats() == b.stats(), (level, i)
        finally:
            a.close()
            b.close()


def test_batches_across_trims(pngb200, budget):
    """peak 0.5 GiB: inflators, host and device contexts and deflators pushed by batch calls, a trim before each call"""
    trimmed, plain = budget(0.5)
    rng = random.Random(8)
    twins = {ctx: dict(z=[], c=[], d=[]) for ctx in (trimmed, plain)}
    infl, ctxs = inflate_streams()[:5], context_files()
    defl = [(pngb200.FORMAT_ZLIB, 9, 15), (pngb200.FORMAT_GZIP, 1, 15)]
    for ctx, t in twins.items():
        t["z"] = [pngb200.Inflator(ctx, fmt) for fmt, _ in infl]
        t["c"] = [Twin(pngb200, ctx, g, k % 2 == 1) for k, (g, _, _) in enumerate(ctxs)]
        t["d"] = [pngb200.Deflator(ctx, *s, online=True) for s in defl]
    streams = [("z", k, s) for k, (_, s) in enumerate(infl)] + [("c", k, idat) for k, (_, idat, _) in enumerate(ctxs)] + \
              [("d", k, text(200_000, 30 + k)) for k in range(len(defl))]
    pos = [0] * len(streams)
    try:
        while any(p <= len(s) for p, (_, _, s) in zip(pos, streams)):
            batch = {"z": [], "c": [], "d": []}
            for i, (kind, k, s) in enumerate(streams):
                if pos[i] > len(s) or rng.random() < 0.2:
                    continue
                n = rng.choice([0, 7, 1000, 20_000, 70_000])
                last = pos[i] + n >= len(s)
                batch[kind].append((k, s[pos[i]:pos[i] + n], rng.random() < 0.5, last))
                pos[i] = pos[i] + n if not last else len(s) + 1
            got = {}
            for ctx, t in twins.items():
                if ctx is trimmed:
                    trimmed.trim()
                sz = pngb200.inflator_push_batch(ctx, [(t["z"][k], p) for k, p, _, _ in batch["z"]])
                if ctx is trimmed:
                    trimmed.trim()
                sc = pngb200.png_context_push_batch(ctx, [(t["c"][k].c, p, od) for k, p, od, _ in batch["c"]])
                if ctx is trimmed:
                    trimmed.trim()
                sd = pngb200.deflator_push_batch(ctx, [(t["d"][k], p, last) for k, p, _, last in batch["d"]])
                got[ctx] = (sz, sc, sd,
                            [inflator_state(t["z"][k]) + (t["z"][k].pull_all(),) for k, _, _, _ in batch["z"]],
                            [t["c"][k].state() for k, _, _, _ in batch["c"]],
                            [(take(t["d"][k], last), t["d"][k].stats()) for k, _, _, last in batch["d"]])
            assert got[trimmed] == got[plain]
    finally:
        for t in twins.values():
            for h in t["z"] + [c.c for c in t["c"]] + t["d"]:
                h.close()
