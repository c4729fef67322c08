"""Cloning the online handles on the H100 (pngb200_clone_batch): Inflator, Deflator, PngContext and PngEncoder are
values, as LZ77.Inflator, LZ77.Deflator, PNG.Context and PNG.Encoder are in the reference.  A handle is cloned after
every push of a seeded stream; every later piece goes into the source, each clone and a never-cloned twin in one batch
call, and after every push each of them must leave what the twin leaves: statuses, error payloads, pulled bytes,
progress, storage, blocks, pieces and stats() (the device bytes a clone holds may be lower).  Clones that are pushed
different data must not see each other's bytes; clones outlive their sources, clone each other, keep sticky errors,
and a batch clone costs at most one launch.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import ctypes as C
import random
import zlib

import numpy as np
import pytest

import deflate_stream as ds
import png_encoder_stream as pes
import pngio
from png_context_cases import GOLDEN, geometry
from test_gpu_deflator_online import take, text
from test_gpu_online_handles import Twin, cut, inflate_streams
from test_gpu_png_context import big_file

pytestmark = pytest.mark.gpu
GiB = 1 << 30


@pytest.fixture
def budget(pngb200):
    """budget(gib) -> a context of its own, after skipping unless `gib` GiB of device memory are free"""
    import torch
    made = []

    def take_(gib: float):
        free, _ = torch.cuda.mem_get_info()
        if free < gib * GiB:
            pytest.skip(f"needs {gib} GiB of free device memory, {free / GiB:.1f} GiB free")
        made.append(pngb200.Context(0))
        return made[-1]

    yield take_
    for c in made:
        c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture
def made(budget):
    """handles a test makes, closed after it whatever happens (before the budget's contexts go)"""
    out = []
    yield out
    close(out)


def storage(c):
    """a PngContext's storage bytes: host, a clone's own device buffer, or a Twin's buffer at an odd address"""
    if c._host is not None:
        return c.storage()
    dev = getattr(c, "_dev", None)
    if dev is not None:
        return dev.cpu().numpy().tobytes()[:c._size]
    return c._twin_buf.cpu().numpy().tobytes()[1:]


def twin_context(pngb200, ctx, g, device):
    t = Twin(pngb200, ctx, g, device)
    t.c._twin_buf = t.buf
    return t.c


# ---- the kinds: make a handle, push one piece into many handles with one call, read a handle's state ----

def inflator_kind(pngb200, fmt):
    def push(ctx, hs, p, i, last):
        return pngb200.inflator_push_batch(ctx, [(h, p) for h in hs])

    def state(h, final):
        return h.error(), h.stats(), h.ctx._lib.pngb200_inflator_available(h.handle), h.pull_all()
    return (lambda ctx: pngb200.Inflator(ctx, fmt)), push, state


def context_kind(pngb200, g, device, overdraw):
    def push(ctx, hs, p, i, last):
        return pngb200.png_context_push_batch(ctx, [(h, p, overdraw and i % 2 == 0) for h in hs])

    def state(h, final):
        return h.error(), h.progress(), storage(h)
    return (lambda ctx: twin_context(pngb200, ctx, g, device)), push, state


def deflator_kind(pngb200, fmt, level, online):
    def push(ctx, hs, p, i, last):
        if online:
            return pngb200.deflator_push_batch(ctx, [(h, p, last) for h in hs])
        return [h.push(p, last) or 0 for h in hs]

    def state(h, final):
        return take(h, final), (h.stats()[:3] if online else ())
    return (lambda ctx: pngb200.Deflator(ctx, fmt, level, 15, chunk_bytes=4000, online=online)), push, state


def encoder_kind(pngb200, fields, w, h, interlaced, level, device):
    def push(ctx, hs, rows, i, last):
        if device:
            import torch
            buf = torch.frombuffer(bytearray(rows), dtype=torch.uint8).cuda() if rows else None
            item = ((buf.data_ptr() if rows else 0, len(rows)), pngb200.MEM_DEVICE)
            return pngb200.png_encoder_push_batch(ctx, [(e, *item) for e in hs])
        return pngb200.png_encoder_push_batch(ctx, [(e, rows) for e in hs])

    def state(e, final):
        return e.pop_all(), e.progress()[:5], e.error()
    return (lambda ctx: pngb200.PngEncoder(ctx, w, h, interlaced=interlaced, level=level, idat_chunk=700, **fields)), \
        push, state


def held(h):
    """the device bytes a handle reports holding, or None for the kinds that report none"""
    if type(h).__name__ == "PngEncoder":
        return h.progress()[5]
    if type(h).__name__ == "Deflator" and h.ctx._lib.pngb200_deflator_stats(h.handle, (C.c_uint64 * 4)()) == 0:
        return h.stats()[3]
    return None


def close(hs):
    for h in hs:
        h.close()


def fork_at_every_push(ctx, kind, pieces, rng):
    """clone after every push (from the source or from an earlier clone); every later piece goes into the source, the
    clones and a twin with one call; after every push each handle must leave what the twin leaves"""
    make, push, state = kind
    twin, src = make(ctx), make(ctx)
    forks = []
    try:
        for i, p in enumerate(pieces):
            last = i == len(pieces) - 1
            hs = [twin, src] + forks
            got = push(ctx, hs, p, i, last)
            want = state(twin, last)
            for k, h in enumerate(hs[1:]):
                assert got[k + 1] == got[0], (i, k)
                assert state(h, last) == want, (i, k)
            assert held(src) == held(twin), i
            origin = rng.choice([src] + forks)
            forks.append(origin.clone())
            if held(origin) is not None:
                assert held(forks[-1]) <= held(origin), i
    finally:
        close([twin, src] + forks)


def test_fork_inflators(pngb200, budget):
    """peak 0.3 GiB: every format with stored blocks, fixed and dynamic blocks, an output that outgrows its buffer and a
    corrupt stream"""
    ctx = budget(0.3)
    rng = random.Random(31)
    for fmt, s in inflate_streams():
        pieces = cut(s, rng, [1, 7, 1000, 20_000, 70_000])
        pieces = pieces[:13] + [b"".join(pieces[13:])]
        fork_at_every_push(ctx, inflator_kind(pngb200, fmt), pieces, rng)


def context_cases():
    out = []
    for il in (False, True):
        png = pngio.parse(big_file(320, 200, il)[1])
        out.append((geometry(png), png.idat, [7, 3000, 20_000]))
    png = pngio.parse(open(f"{GOLDEN}/pngsuite/z00n2c08.png", "rb").read())
    out.append((geometry(png), png.idat, [7, 300, 1000]))
    return out


def test_fork_contexts(pngb200, budget):
    """peak 0.3 GiB: host and device storage, plain and Adam7, with and without overdraw"""
    ctx = budget(0.3)
    rng = random.Random(32)
    for device in (False, True):
        for overdraw in (False, True):
            for g, idat, sizes in context_cases():
                pieces = cut(idat, rng, sizes)
                pieces = pieces[:11] + [b"".join(pieces[11:])]
                fork_at_every_push(ctx, context_kind(pngb200, g, device, overdraw), pieces, rng)


def test_fork_deflators(pngb200, budget):
    """peak 0.5 GiB: online levels 0, 4, 9 and 13 and a buffered deflator"""
    ctx = budget(0.5)
    rng = random.Random(33)
    for fmt, level, online in ((ds.ZLIB, 0, True), (ds.GZIP, 4, True), (ds.ZLIB, 9, True), (ds.IOS, 13, True),
                               (ds.ZLIB, 9, False)):
        data = text(30_000 if level == 13 else 200_000, level)
        pieces = cut(data, rng, [1, 700, 4097, 30_000])[:12]
        pieces[-1] = data[sum(len(p) for p in pieces[:-1]):]
        fork_at_every_push(ctx, deflator_kind(pngb200, fmt, level, online), pieces, rng)


def test_fork_encoders(pngb200, budget, orc):
    """peak 0.3 GiB: host and device rows, plain and Adam7"""
    ctx = budget(0.3)
    rng = random.Random(34)
    fields, w, h = dict(color=6, depth=8), 120, 40
    px = np.random.default_rng(5).integers(0, 40, w * h * 4, dtype=np.uint8).tobytes()
    for device in (False, True):
        for interlaced in (False, True):
            sched = pes.schedule(h, [3, 0, 5, 1])
            rows, at = [], 0
            for n in sched:
                rows.append(px[at * w * 4:(at + n) * w * 4])
                at += n
            fork_at_every_push(ctx, encoder_kind(pngb200, fields, w, h, interlaced, 6, device), rows, rng)


def diverge(ctx, kind, pieces, other, k, in_clone):
    """push pieces[:k], clone, then `pieces` into one handle and `other` into the other (the clone when `in_clone`),
    each beside a twin that never saw a clone; after every push into one handle both handles equal their twins, byte for
    byte: pulled bytes, blocks, pieces and storage"""
    make, push, state = kind
    twin_a, twin_b, src = make(ctx), make(ctx), make(ctx)
    hs = [twin_a, twin_b, src]
    try:
        for i, p in enumerate(pieces[:k]):
            push(ctx, hs, p, i, False)
        hs.append(src.clone())
        a, b = (src, hs[3]) if in_clone else (hs[3], src)
        for i in range(k, max(len(pieces), len(other))):
            for h, twin, seq in ((a, twin_a, pieces), (b, twin_b, other)):
                if i >= len(seq):
                    continue
                last = i == len(seq) - 1
                got = push(ctx, [twin, h], seq[i], i, last)
                assert got[0] == got[1], i
                assert state(h, last) == state(twin, last), i
                o, ot = (b, twin_b) if h is a else (a, twin_a)
                assert state(o, False) == state(ot, False), i
    finally:
        close(hs)


def corrupt(pieces, k):
    """pieces[k:] with a byte flipped in the first of them and in the stream's last byte (its checksum)"""
    out = [bytearray(p) for p in pieces]
    out[k][len(out[k]) // 2] ^= 0x5A
    out[-2 if not out[-1] else -1][-1] ^= 0xFF
    return [bytes(p) for p in out]


def test_divergence_and_aliasing(pngb200, budget):
    """peak 0.3 GiB: after the clone one handle takes a corrupt continuation and the other the true one (and the
    reverse), or two different streams; each finishes equal to a twin that took the same bytes, and no push into one
    changes what the other returns"""
    ctx = budget(0.3)
    rng = random.Random(35)
    g, idat, _ = context_cases()[1]
    pieces = cut(idat, rng, [5000, 20_000])
    for device in (False, True):
        for in_clone in (False, True):
            for k in (1, len(pieces) // 2):
                diverge(ctx, context_kind(pngb200, g, device, False), pieces, corrupt(pieces, k), k, in_clone)
    fmt, s = inflate_streams()[4]
    pieces = cut(s, rng, [1000, 20_000])
    for in_clone in (False, True):
        diverge(ctx, inflator_kind(pngb200, fmt), pieces, corrupt(pieces, 2), 2, in_clone)
    data, more = text(100_000, 3), text(100_000, 4)
    pieces, other = cut(data, rng, [700, 9000]), cut(data[:20_000] + more, rng, [700, 9000])
    diverge(ctx, deflator_kind(pngb200, ds.ZLIB, 9, True), pieces, other, 1, True)
    fields, w, h = dict(color=0, depth=8), 100, 30
    px = [np.random.default_rng(s).integers(0, 256, w * h, dtype=np.uint8).tobytes() for s in (1, 2)]
    rows = [[p[y * w * 3:(y + 1) * w * 3] for y in range(10)] for p in px]
    rows[1][:2] = rows[0][:2]
    diverge(ctx, encoder_kind(pngb200, fields, w, h, True, 4, False), rows[0], rows[1], 2, True)


def test_lifetimes(pngb200, budget, made):
    """peak 0.3 GiB: a clone outlives its source, a clone of a clone, clones of terminal handles, of handles with a
    sticky error and of an encoder with pieces not popped, and ctx.trim() between a clone and the next push"""
    ctx = budget(0.3)
    rng = random.Random(36)
    g, idat, _ = context_cases()[0]
    pieces = [p for p in cut(idat, rng, [3000, 20_000]) if p]
    for device in (False, True):
        twin, src = twin_context(pngb200, ctx, g, device), twin_context(pngb200, ctx, g, device)
        made += [twin, src]
        for p in pieces[:3]:
            twin.push(p), src.push(p)
        c1 = src.clone()
        src.close()
        ctx.trim()
        c2 = c1.clone()
        made += [c1, c2]
        for p in pieces[3:]:
            twin.push(p), c1.push(p), c2.push(p)
            assert (c1.error(), c1.progress(), storage(c1)) == (twin.error(), twin.progress(), storage(twin))
            assert (c2.error(), c2.progress(), storage(c2)) == (twin.error(), twin.progress(), storage(twin))
        c3 = c2.clone()   # terminal
        made.append(c3)
        for c in (twin, c3):
            with pytest.raises(pngb200.PNGB200Error) as e:
                c.push(b"x")
            assert e.value.status == pngb200.ERR_PNG_EXTRANEOUS_COMPRESSED_DATA
        assert (c3.progress(), storage(c3)) == (twin.progress(), storage(twin))
        close([twin, c1, c2, c3])
    # an inflator with a sticky error, and a terminal one
    fmt, s = inflate_streams()[-1]
    z = pngb200.Inflator(ctx, fmt)
    made.append(z)
    with pytest.raises(pngb200.PNGB200Error) as e:
        z.push(s)
    y = z.clone()
    made.append(y)
    assert y.error() == z.error() and y.error()[0] == e.value.status
    with pytest.raises(pngb200.PNGB200Error):
        y.push(b"more")
    fmt, s = inflate_streams()[3]
    t = pngb200.Inflator(ctx, fmt)
    made.append(t)
    assert t.push(s) == pngb200.OK
    u = t.clone()
    made.append(u)
    assert u.push(b"ignored") == pngb200.OK and u.pull_all() == t.pull_all() == zlib.decompress(s)
    close([z, y, t, u])
    # an encoder with pieces not popped: each handle pops its own copy
    fields, w, h = dict(color=0, depth=8), 200, 60
    px = np.random.default_rng(9).integers(0, 256, w * h, dtype=np.uint8).tobytes()
    e = pngb200.PngEncoder(ctx, w, h, level=4, idat_chunk=100, **fields)
    made.append(e)
    e.push(px[:w * 30])
    f = e.clone()
    made.append(f)
    ctx.trim()
    first = e.pop_all()
    assert len(first) > 1 and f.pop_all() == first and f.pop_all() == []
    e.push(px[w * 30:]), f.push(px[w * 30:])
    a, b = e.pop_all(), f.pop_all()
    assert a == b and a[-1][4:8] == b"IEND"
    ((st, whole),) = pngb200.png_encode_batch(ctx, [dict(storage=px, width=w, height=h, **fields)], 4, 100)
    assert st == 0 and b"".join(first + a) == whole
    d = f.clone()   # after IEND
    made.append(d)
    assert d.pop_all() == [] and d.progress()[:5] == f.progress()[:5]
    close([e, f, d])
    # a deflator after `last`
    z = pngb200.Deflator(ctx, ds.ZLIB, 9, online=True)
    made.append(z)
    z.push(b"abc" * 1000, last=True)
    y = z.clone()
    made.append(y)
    assert take(y, True) == take(z, True)
    with pytest.raises(pngb200.PNGB200Error):
        y.push(b"x")
    close([z, y])


def test_large_state(pngb200, budget, made, orc):
    """peak 2 GiB: a level-8 deflator cloned mid-block near DF_GRAPH_CAP in the 6 MB stream, and an 8K Adam7 context
    cloned halfway; both branches finish equal to the reference's output"""
    ctx = budget(2)
    data = text(6 << 20, 77)
    cuts = ds.cuts(len(data), [65544])
    z = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, level=8, online=True)
    made.append(z)
    out = []
    for a, b in cuts[:len(cuts) * 3 // 4]:
        z.push(data[a:b])
        out += take(z, False)
    y = z.clone()
    made.append(y)
    assert y.stats()[:3] == z.stats()[:3] and y.stats()[3] <= z.stats()[3]
    branches = []
    for h in (z, y):
        got = list(out)
        for a, b in cuts[len(cuts) * 3 // 4:]:
            h.push(data[a:b])
            got += take(h, False)
        h.push(b"", last=True)
        branches.append(b"".join(got + take(h, True)))
    assert branches[0] == branches[1] == orc.deflate(data, 8)
    close([z, y])
    img, file = big_file(7680, 4320, True)
    png = pngio.parse(file)
    g = geometry(png)
    chunks = pngio.idat_chunks(file)
    src = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], True, g["standard"])
    made.append(src)
    for c in chunks[:len(chunks) // 2]:
        src.push(c)
    clone = src.clone()
    made.append(clone)
    for c in chunks[len(chunks) // 2:]:
        src.push(c)
        clone.push(c)
    src.end(), clone.end()
    assert src.storage() == clone.storage() == img
    close([src, clone])


def test_batch_and_launches(pngb200, budget, made):
    """peak 0.5 GiB: one clone_batch of 64 mixed items equals the same clones made one at a time; a call makes at most
    one launch, and none when no item holds device bytes"""
    ctx = budget(0.5)
    rng = random.Random(37)
    g, idat, _ = context_cases()[1]
    srcs = []
    for i in range(64):
        kind = i % 4
        if kind == 0:
            fmt, s = inflate_streams()[i % 5]
            h = pngb200.Inflator(ctx, fmt)
            h.push(s[: len(s) // 3])
        elif kind == 1:
            h = pngb200.Deflator(ctx, ds.ZLIB, rng.choice([0, 4, 9]), online=i % 8 != 1)
            h.push(text(20_000, i))
        elif kind == 2:
            h = twin_context(pngb200, ctx, g, i % 8 == 2)
            h.push(idat[:5000 + 100 * i])
            h.rest = idat[5000 + 100 * i:]
        else:
            h = pngb200.PngEncoder(ctx, 64, 16, color=2, depth=8, level=6, idat_chunk=300)
            h.push(bytes(range(256)) * 3 * 4)
        srcs.append(h)
    made += srcs
    n0 = ctx.launches
    batch = pngb200.clone_batch(ctx, srcs)
    made += batch
    assert ctx.launches - n0 <= 1
    alone = [s.clone() for s in srcs]
    made += alone

    def state(h, src):
        if isinstance(h, pngb200.Inflator):
            return h.error(), h.stats(), h.pull_all()
        if isinstance(h, pngb200.Deflator):
            h.push(b"tail", last=True)
            return take(h, True)
        if isinstance(h, pngb200.PngContext):
            h.push(src.rest)
            return h.error(), h.progress(), storage(h)
        return h.pop_all(), h.progress()[:5]
    for a, b, src in zip(batch, alone, srcs):
        assert state(a, src) == state(b, src)
    close(batch + alone + srcs)
    # all-host items: fresh handles and buffered deflators
    fresh = [pngb200.Inflator(ctx, 0), pngb200.Deflator(ctx, ds.ZLIB, 9)]
    fresh[1].push(b"host bytes")
    made += fresh
    n0 = ctx.launches
    made += pngb200.clone_batch(ctx, fresh)
    assert ctx.launches == n0 and ctx.clone_stats() == (0, len(b"host bytes"))
    # the bytes a call copies: an inflator's input and output
    fmt, s = inflate_streams()[3]
    z = pngb200.Inflator(ctx, fmt)
    made.append(z)
    z.push(s)
    made.append(z.clone())
    assert ctx.clone_stats()[0] == len(s) + len(zlib.decompress(s))


def test_rejections(pngb200, budget, made):
    """peak 0.2 GiB: every rejection leaves every clone NULL and the sources usable"""
    import ctypes as C
    import torch
    ctx, other = budget(0.2), budget(0)
    L = ctx._lib
    g, idat, _ = context_cases()[0]
    host = pngb200.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"])
    dev = twin_context(pngb200, ctx, g, True)
    z = pngb200.Inflator(ctx, 0)
    foreign = pngb200.Inflator(other, 0)
    made += [host, dev, z, foreign]
    size = host._size
    buf = torch.empty(size, dtype=torch.uint8, device="cuda")
    own = C.create_string_buffer(size)

    def call(items):
        descs = (pngb200.CloneDesc * max(len(items), 1))()
        for d, it in zip(descs, items):
            for k, v in it.items():
                setattr(d, k, v)
            d.clone = 12345
        rc = L.pngb200_clone_batch(ctx.handle, descs, len(items))
        assert all(not descs[i].clone for i in range(len(items)))
        return rc

    bad = pngb200.ERR_BAD_ARGUMENT
    assert L.pngb200_clone_batch(None, None, 0) == bad
    assert L.pngb200_clone_batch(ctx.handle, None, 1) == bad
    ok = dict(inflator=z.handle)
    assert call([ok, {}]) == bad
    assert call([ok, dict(inflator=z.handle, deflator=z.handle)]) == bad
    assert call([ok, dict(inflator=foreign.handle)]) == bad
    assert call([ok, dict(context=host.handle, pixels=None, pixels_cap=size)]) == bad
    assert call([ok, dict(context=host.handle, pixels=C.addressof(own), pixels_cap=size - 1)]) == bad
    assert call([ok, dict(context=host.handle, pixels=host._addr + 1, pixels_cap=size)]) == bad
    dev_addr = dev._twin_buf.data_ptr() + 1
    assert call([ok, dict(context=dev.handle, pixels=dev_addr - size + 1, pixels_cap=size)]) == bad
    # a pending decode batch
    from oracle import oracle
    img = bytes(np.random.default_rng(1).integers(0, 256, 64 * 64 * 4, dtype=np.uint8))
    zs = zlib.compress(oracle.png_filter(img, 64, 64, 32, 8), 6)
    descs = (pngb200.ImageDesc * 1)()
    out = C.create_string_buffer(len(img))
    descs[0].idat, descs[0].idat_len = C.cast(C.c_char_p(zs), C.c_void_p), len(zs)
    descs[0].width, descs[0].height, descs[0].volume, descs[0].depth = 64, 64, 32, 8
    descs[0].pixels, descs[0].pixels_cap = C.addressof(out), len(img)
    assert L.pngb200_decode_batch_enqueue(ctx.handle, descs, 1, pngb200.MEM_HOST) == 0
    assert call([ok]) == bad
    assert L.pngb200_decode_batch_finish(ctx.handle, descs, 1) == 0
    assert descs[0].status == 0 and out.raw == img
    # Python: host storage is always the clone's own
    with pytest.raises(pngb200.PNGB200Error):
        pngb200.clone_batch(ctx, [(host, (C.addressof(own), size))])
    # the sources are still usable and can be cloned
    host.push(idat[:4000]), dev.push(idat[:4000]), z.push(zlib.compress(b"abc"))
    clones = pngb200.clone_batch(ctx, [host, (dev, (buf.data_ptr(), size)), z])
    made += clones
    assert storage(clones[0]) == storage(host) and buf.cpu().numpy().tobytes() == storage(dev)
    assert clones[2].pull_all() == z.pull_all() == b"abc"
    close([foreign])
