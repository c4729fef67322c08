"""Batch online decoding on the H100 (pngb200_png_context_push_batch, pngb200_inflator_push_batch): many contexts and
inflators pushed in one call.  Every item must show what the same push made alone shows: status, error payload,
progress, storage, available and pulled bytes and work counters; the launches of a call must not grow with the number of
items; and call-level errors touch no item.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import random
import zlib

import numpy as np
import pytest

import pngio
from oracle import oracle
from png_context_cases import OracleContext, geometry, goldens
from test_gpu_inflate_resume import FORMATS, long_block
from test_gpu_png_context import big_file

pytestmark = pytest.mark.gpu
GiB = 1 << 30
GOLDENS = goldens()
EXTRANEOUS_COMPRESSED = -49
ASSIGN_BOUND = 1 + 7          # unfilter + assign launches of one call, beyond the inflator's
INFLATE_BOUND = 2 + 2         # ring + serial, then the checksum pair, per round


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


class Item:
    """a GPU context, host storage or device storage at an odd address, and its oracle twin"""

    def __init__(self, pngb200, ctx, g, device):
        self.g, self.buf = g, None
        self.size = oracle.storage_size(g["w"], g["h"], g["volume"])
        if device:
            import torch
            self.buf = torch.full((self.size + 1,), 0x5A, dtype=torch.uint8, device="cuda")
            self.gpu = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"],
                                          (self.buf.data_ptr() + 1, self.size))
        else:
            self.gpu = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"])
        self.ref = OracleContext(**g)

    def storage(self):
        if self.buf is None:
            return self.gpu.storage()
        return bytes(self.buf.cpu().numpy().tobytes()[1:1 + self.size])

    def check(self, st, want, tag):
        assert st == want, tag
        assert self.gpu.progress() == self.ref.progress(), tag
        if st < 0 and st != EXTRANEOUS_COMPRESSED:
            assert self.gpu.error()[1:] == self.ref.error()[1:], tag
        assert self.storage() == self.ref.storage(), tag

    def close(self):
        self.gpu.close()
        self.ref.close()


def run_goldens(pngb200, ctx, piece_lists):
    items = [Item(pngb200, ctx, geometry(pngio.parse(data)), i % 3 == 2) for i, (_, data) in enumerate(GOLDENS)]
    try:
        rounds = max(len(p) for p in piece_lists)
        for r in range(rounds + 1):
            batch = []
            for i, (it, pieces) in enumerate(zip(items, piece_lists)):
                if r < len(pieces):
                    batch.append((it, pieces[r], (i + r) % 2 == 1))
                elif r == len(pieces):
                    batch.append((it, b"", False))   # one empty push after the last piece
            sts = pngb200.png_context_push_batch(ctx, [(it.gpu, p, od) for it, p, od in batch])
            for (it, p, od), st in zip(batch, sts):
                it.check(st, it.ref.push(p, od), (r, it.g))
        for it in items:
            assert it.gpu.progress()[3] == 1
    finally:
        for it in items:
            it.close()


def test_every_golden_in_one_batch(pngb200, budget):
    """peak 0.5 GiB: one context per golden, round r pushing each one's r-th IDAT chunk, then its 7-byte pieces (4 099
    for the colour goldens); after every round every context matches its oracle"""
    ctx = budget(0.5)
    run_goldens(pngb200, ctx, [pngio.idat_chunks(data) for _, data in GOLDENS])
    sevens = []
    for _, data in GOLDENS:
        idat = pngio.parse(data).idat
        step = 7 if len(idat) <= 16384 else 4099
        sevens.append([idat[i:i + step] for i in range(0, len(idat), step)])
    run_goldens(pngb200, ctx, sevens)


def test_terminal_and_errored_items_cost_no_launch(pngb200, budget):
    """peak 0.1 GiB: a finished context answers -49 on the host, with no launch"""
    ctx = budget(0.1)
    name, data = GOLDENS[0]
    it = Item(pngb200, ctx, geometry(pngio.parse(data)), False)
    try:
        assert pngb200.png_context_push_batch(ctx, [(it.gpu, pngio.parse(data).idat, False)]) == [0]
        n = ctx.launches
        assert pngb200.png_context_push_batch(ctx, [(it.gpu, b"", False)]) == [EXTRANEOUS_COMPRESSED]
        assert ctx.launches == n
    finally:
        it.close()


def _inflator_state(z):
    return (z.error(), z.stats(), z.ctx._lib.pngb200_inflator_available(z.handle))


def test_batch_equals_singles(pngb200, budget):
    """peak 1 GiB: a seeded schedule of random subsets and random piece sizes, some across 64 KiB so that ring and
    serial jobs share a round; a twin set of handles takes the same pushes one at a time"""
    ctx = budget(1)
    rng = random.Random(11)
    files = [big_file(640, 360, il)[1] for il in (False, True)] + [d for n, d in GOLDENS if n.startswith("colour/")][:4]
    streams = []
    for f in files:
        png = pngio.parse(f)
        streams.append((geometry(png), png.idat))
    raw = [(fmt, (lambda c: c.compress(bytes(np.random.default_rng(fmt).integers(0, 8, 400_000, dtype=np.uint8))) + c.flush())(
        zlib.compressobj(9, zlib.DEFLATED, wb))) for fmt, wb in FORMATS.values()]
    pairs, infl = [], []
    for g, idat in streams:
        mk = lambda: pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"])
        pairs.append([mk(), mk(), idat, 0, len(pairs) % 2 == 0])
    for fmt, s in raw:
        infl.append([pngb200.Inflator(ctx, fmt), pngb200.Inflator(ctx, fmt), s, 0])
    try:
        for rnd in range(400):
            live_c = [p for p in pairs if p[3] <= len(p[2])]
            live_i = [p for p in infl if p[3] <= len(p[2])]
            if not live_c and not live_i:
                break
            cb, ib = [], []
            for p in live_c + live_i:
                if rng.random() < 0.3:
                    continue
                n = rng.choice([0, 1, 7, 1000, 20_000, 70_000, 150_000])
                piece = p[2][p[3]:p[3] + n]
                p[3] += max(n, 1)
                (cb if p in live_c else ib).append((p, piece))
            od = rng.random() < 0.5
            sts = pngb200.png_context_push_batch(ctx, [(p[0], piece, od) for p, piece in cb])
            for (p, piece), st in zip(cb, sts):
                try:
                    p[1].push(piece, od)
                    one = 0
                except pngb200.PNGB200Error as e:
                    one = e.status
                assert st == one, rnd
                assert p[0].progress() == p[1].progress() and p[0].error() == p[1].error(), rnd
                assert p[0].storage() == p[1].storage(), rnd
            sts = pngb200.inflator_push_batch(ctx, [(p[0], piece) for p, piece in ib])
            for (p, piece), st in zip(ib, sts):
                try:
                    one = p[1].push(piece)
                except pngb200.PNGB200Error as e:
                    one = e.status
                assert st == one and _inflator_state(p[0]) == _inflator_state(p[1]), rnd
                if rng.random() < 0.3:
                    k = rng.randrange(0, p[0].ctx._lib.pngb200_inflator_available(p[0].handle) + 1)
                    assert p[0].pull(k) == p[1].pull(k)
        for p in infl:
            assert p[0].pull_all() == p[1].pull_all()
    finally:
        for p in pairs + infl:
            p[0].close()
            p[1].close()


def test_inflator_batch(pngb200, budget):
    """peak 1 GiB: zlib, ios and gzip streams with stored blocks, a 16 MiB dynamic block cut into 65 544-byte pushes, an
    item whose output has to grow while the others do not, a corrupt item whose error stays its own, and a terminal
    item answered with no work; every item against oracle.inflate of what it was pushed"""
    ctx = budget(1)
    rng = np.random.default_rng(5)
    plain = rng.integers(0, 256, 300_000, dtype=np.uint8).tobytes()
    streams = []   # (format, stream, plain)
    for fmt, wb in FORMATS.values():
        c = zlib.compressobj(0 if fmt == 1 else 6, zlib.DEFLATED, wb)   # level 0: stored blocks
        streams.append((fmt, c.compress(plain) + c.flush(), plain))
    big, big_plain, _ = long_block("dynamic").finish("zlib")
    streams.append((0, big, big_plain))
    streams.append((0, zlib.compress(bytes(3_000_000), 9), bytes(3_000_000)))   # 3 KB in, 3 MB out: the output grows
    bad = bytearray(zlib.compress(plain[:50_000], 6))
    bad[len(bad) // 2] ^= 0x5A
    streams.append((0, bytes(bad), None))
    done = pngb200.Inflator(ctx, 0)
    assert done.push(zlib.compress(b"x" * 100)) == 0
    hs = [pngb200.Inflator(ctx, fmt) for fmt, _, _ in streams]
    pos, got = [0] * len(streams), [b""] * len(streams)
    try:
        while any(p < len(s) for p, (_, s, _) in zip(pos, streams)):
            items, idx = [(done, b"more")], []
            for k, (fmt, s, _) in enumerate(streams):
                if pos[k] < len(s):
                    items.append((hs[k], s[pos[k]:pos[k] + (65544 if k != 4 else len(s))]))
                    idx.append(k)
                    pos[k] += len(items[-1][1])
            n, stats = ctx.launches, done.stats()
            sts = pngb200.inflator_push_batch(ctx, items)
            assert sts[0] == 0 and done.stats() == stats
            for k, st in zip(idx, sts[1:]):
                fmt, s, full = streams[k]
                got[k] += hs[k].pull_all()
                if k == 3:   # 16 MiB: the handle's output is the plain text's prefix, complete at the end
                    assert st == (0 if pos[k] == len(s) else 1) and big_plain.startswith(got[k]), k
                    continue
                want = oracle.inflate(s[:pos[k]], fmt, 1 << 23)
                assert st == want[0], (k, st, want[0])
                assert want[1].startswith(got[k]), k   # a stored block is released once all of it has arrived
                if st < 0:
                    assert hs[k].error()[1:] == (want[2].a, want[2].b), k
                    pos[k] = len(s)
        for k, (_, _, full) in enumerate(streams):
            assert full is None or got[k] == full, k
        assert hs[-1].error()[0] < 0
    finally:
        done.close()
        for h in hs:
            h.close()


def test_call_level_rejections(pngb200, budget):
    """peak 0.1 GiB: a duplicate handle, a handle of another ctx, data NULL with n > 0 and a pending decode batch give
    BAD_ARGUMENT with no item touched; count 0 is OK; an inflator batch works while a decode batch is pending"""
    import ctypes as C
    ctx = budget(0.1)
    other = pngb200.Context(0)
    _, data = GOLDENS[0]
    g = geometry(pngio.parse(data))
    idat = pngio.parse(data).idat
    a = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"])
    b = pngb200.PngContext(other, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"])
    z = pngb200.Inflator(ctx)
    try:
        before = (a.progress(), a.storage())
        for items in ([(a, idat, False), (a, idat, False)], [(a, idat, False), (b, idat, False)]):
            with pytest.raises(pngb200.PNGB200Error) as e:
                pngb200.png_context_push_batch(ctx, items)
            assert e.value.status == pngb200.ERR_BAD_ARGUMENT
            assert (a.progress(), a.storage()) == before
        d = (pngb200.PngPushDesc * 1)()
        d[0].context, d[0].data, d[0].n = a.handle, None, 5
        assert ctx._lib.pngb200_png_context_push_batch(ctx.handle, d, 1) == pngb200.ERR_BAD_ARGUMENT
        assert ctx._lib.pngb200_png_context_push_batch(ctx.handle, d, 0) == 0
        assert ctx._lib.pngb200_inflator_push_batch(ctx.handle, None, 0) == 0
        assert (a.progress(), a.storage()) == before
        with pytest.raises(pngb200.PNGB200Error):
            pngb200.inflator_push_batch(ctx, [(z, b"ab"), (z, b"cd")])
        # a pending decode batch
        img = bytes(np.random.default_rng(1).integers(0, 256, 64 * 64 * 4, dtype=np.uint8))
        zs = zlib.compress(oracle.png_filter(img, 64, 64, 32, 8), 6)
        descs = (pngb200.ImageDesc * 1)()
        out = C.create_string_buffer(len(img))
        descs[0].idat, descs[0].idat_len = C.cast(C.c_char_p(zs), C.c_void_p), len(zs)
        descs[0].width, descs[0].height, descs[0].volume, descs[0].depth = 64, 64, 32, 8
        descs[0].pixels, descs[0].pixels_cap = C.addressof(out), len(img)
        assert ctx._lib.pngb200_decode_batch_enqueue(ctx.handle, descs, 1, pngb200.MEM_HOST) == 0
        with pytest.raises(pngb200.PNGB200Error) as e:
            pngb200.png_context_push_batch(ctx, [(a, idat, False)])
        assert e.value.status == pngb200.ERR_BAD_ARGUMENT and (a.progress(), a.storage()) == before
        s = zlib.compress(b"streaming while a batch is pending" * 100)
        assert pngb200.inflator_push_batch(ctx, [(z, s)]) == [0]
        assert z.pull_all() == b"streaming while a batch is pending" * 100
        assert ctx._lib.pngb200_decode_batch_finish(ctx.handle, descs, 1) == 0
        assert descs[0].status == 0 and out.raw == img
    finally:
        a.close()
        b.close()
        z.close()
        other.close()


def test_launches_do_not_grow_with_the_batch(pngb200, budget):
    """peak 4 GiB: 1, 8 and 64 contexts of one 1080p file pushed by its 65 544-byte chunks: launches per round stay
    within the header's bound and are the same for 64 contexts as for 1"""
    ctx = budget(4)
    img, f = big_file(1920, 1080, False)
    chunks = pngio.idat_chunks(f)
    per_n = {}
    for n in (1, 8, 64):
        cs = [pngb200.PngContext(ctx, 1920, 1080, 32, 8, False) for _ in range(n)]
        counts = []
        try:
            for ch in chunks:
                before = ctx.launches
                assert pngb200.png_context_push_batch(ctx, [(c, ch, True) for c in cs]) == [0] * n
                counts.append(ctx.launches - before)
            for c in cs:
                assert c.storage() == img
        finally:
            for c in cs:
                c.close()
        assert max(counts) <= INFLATE_BOUND + ASSIGN_BOUND
        per_n[n] = counts
    assert per_n[1] == per_n[8] == per_n[64]


def test_large_batches(pngb200, budget):
    """peak 12 GiB: 16 x 1080p (plain and Adam7, host and device storage) and 2 x 8K RGBA8 in one batch, pushed by
    65 544-byte chunks; the oracle at sampled rounds, and png_decode_batch's storage at the end"""
    import torch
    ctx = budget(12)
    files = [big_file(1920, 1080, il) for il in (False, True)] + [big_file(7680, 4320, il) for il in (False, True)]
    specs = [(1920, 1080, k % 2 == 1, k % 4 >= 2) for k in range(16)] + [(7680, 4320, False, False), (7680, 4320, True, False)]
    for img, f in files:
        (dec,) = pngb200.png_decode_batch(ctx, [f])
        assert dec.status == 0 and dec.storage == img
    items = []
    for w, h, il, dev in specs:
        img, f = files[(2 if w > 4000 else 0) + il]
        buf = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda") if dev else None
        c = pngb200.PngContext(ctx, w, h, 32, 8, il, 0, (buf.data_ptr(), w * h * 4) if dev else None)
        items.append(dict(c=c, buf=buf, img=img, chunks=pngio.idat_chunks(f), ref=OracleContext(w, h, 32, 8, il) if w < 4000 else None,
                          pending=b""))
    try:
        rounds = max(len(it["chunks"]) for it in items)
        sample = set(np.linspace(0, rounds - 1, 4).astype(int).tolist())
        for r in range(rounds):
            batch = [it for it in items if r < len(it["chunks"])]
            sts = pngb200.png_context_push_batch(ctx, [(it["c"], it["chunks"][r], r % 2 == 0) for it in batch])
            assert sts == [0] * len(batch)
            for it in batch:
                if it["ref"] is None:
                    continue
                it["pending"] += it["chunks"][r]
                if r in sample or r == len(it["chunks"]) - 1:
                    assert it["ref"].push(it["pending"], r % 2 == 0) == 0
                    it["pending"] = b""
                    got = it["c"].storage() if it["buf"] is None else bytes(it["buf"].cpu().numpy().tobytes())
                    assert it["c"].progress()[:4] == it["ref"].progress()[:4], r
                    assert got == it["ref"].storage(), r
        for it in items:
            it["c"].end()
            got = it["c"].storage() if it["buf"] is None else bytes(it["buf"].cpu().numpy().tobytes())
            assert got == it["img"]
    finally:
        for it in items:
            it["c"].close()
            if it["ref"] is not None:
                it["ref"].close()
