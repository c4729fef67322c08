"""The online PNG encoder (pngb200_png_encoder_*) on the GPU: after every push the pieces pop() hands out are exactly
the restatement's (tests/png_encoder_stream.py, PNG.Encoder.pull with rows arriving over time), and joined they are
pngb200_png_encode_batch's file -- the committed level-9 outputs byte for byte.  Device rows read in place give the
same pieces; a batch push is the same pushes made alone, refuses bad calls whole and keeps its launch bound; a wide
image pushed in bands keeps the handle's device memory flat."""
from __future__ import annotations

import ctypes as C
import os
import random
import zlib

import numpy as np
import pytest

import corpus
import png_encoder_stream as pes
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

KEPT = sorted(f[4:] for f in os.listdir(os.path.join(GOLDEN, "encode")) if f.startswith("out-"))
FORMATS = ((dict(color=6, depth=8, bgr=True), 5, 4), (dict(color=2, depth=8, bgr=True, key=(3, 2, 1)), 4, 4),
           (dict(color=0, depth=4, key=(9,)), 7, 3), (dict(color=2, depth=16, key=(1, 2, 3)), 3, 3),
           (dict(color=3, depth=2, palette=bytes([1, 2, 3, 255, 4, 5, 6, 7, 8, 9, 10, 255])), 9, 2),
           (dict(color=6, depth=16), 64, 48), (dict(color=4, depth=8), 33, 17), (dict(color=0, depth=1), 9, 9))
MAX_LAUNCHES = 3   # filter, deflate, CRC-32 (pngb200.h, pngb200_png_encoder_push_batch)


def noise(fields, w, h, seed):
    rng = np.random.default_rng(seed)
    top = 3 if fields["color"] == 3 else (1 << min(fields["depth"], 8))
    n = w * h * pes.CHANNELS[fields["color"]] * (2 if fields["depth"] == 16 else 1)
    return rng.integers(0, top, n, dtype=np.uint8).tobytes()


def bands(storage, h, sched):
    """the storage bytes of each push of `sched`"""
    row = len(storage) // h
    out, at = [], 0
    for n in sched:
        out.append(storage[at * row: (at + n) * row])
        at += n
    return out


def stream(pngb200, ctx, storage, w, h, fields, interlaced, level, chunk, sched, orc=None):
    """push `sched` through one encoder; the pieces after each push (and, with `orc`, check them against the
    restatement's as they come)"""
    e = pngb200.PngEncoder(ctx, w, h, interlaced=interlaced, level=level, idat_chunk=chunk, **fields)
    want = pes.pieces(orc, storage, w, h, fields, interlaced, level, chunk or 65544, sched) if orc else None
    got = []
    for k, rows in enumerate(bands(storage, h, sched)):
        e.push(rows)
        got.append(e.pop_all())
        if want is not None:
            assert got[-1] == want[k], (level, chunk, interlaced, k, [len(p) for p in got[-1]], [len(p) for p in want[k]])
    p = e.progress()
    assert p[0] == h and p[4] == 1 and p[3] == sum(c[4:8] == b"IDAT" for g in got for c in g)
    e.close()
    return got


def baseline(orc, name):
    info, storage = orc.png_decompress(open(os.path.join(GOLDEN, "encode", "in-" + name), "rb").read())
    assert info.status == 0
    return storage, info.width, info.height, info.fields(), bool(info.interlaced)


@pytest.mark.parametrize("name", KEPT)
def test_level9_outputs_in_every_schedule(pngb200, ctx, orc, name):
    storage, w, h, fields, interlaced = baseline(orc, name)
    out = open(os.path.join(GOLDEN, "encode", "out-" + name), "rb").read()
    for kind in ("rows", 7, "all"):
        got = stream(pngb200, ctx, storage, w, h, fields, interlaced, 9, 0, pes.schedule(h, kind), orc)
        assert b"".join(b"".join(g) for g in got) == out, kind
        if kind == "rows" and sum(c[4:8] == b"IDAT" for g in got for c in g) > 2:
            assert next(i for i, g in enumerate(got) if len(g) > (i == 0)) < h - 1


@pytest.mark.parametrize("k", range(len(FORMATS)))
def test_formats_levels_and_chunks(pngb200, ctx, orc, k):
    fields, w, h = FORMATS[k]
    storage = noise(fields, w, h, 20 + k)
    for interlaced in (False, True):
        for level in (0, 4, 9, 13):
            for chunk in (16, 65544):
                got = stream(pngb200, ctx, storage, w, h, fields, interlaced, level, chunk, pes.schedule(h, [2, 0, 5, 1]), orc)
                ((st, whole),) = pngb200.png_encode_batch(ctx, [dict(storage=storage, width=w, height=h,
                                                                     interlaced=interlaced, **fields)], level, chunk)
                assert st == 0 and b"".join(b"".join(g) for g in got) == whole, (interlaced, level, chunk)


def test_scanline_ends_on_both_sides_of_the_trigger(pngb200, ctx, orc):
    """scanlines of 4095, 4096 and 4097 filtered bytes pushed in bands: each scanline end decides a compression pass"""
    for w in (4094, 4095, 4096):
        fields = dict(color=0, depth=8)
        px = np.ascontiguousarray(corpus.make("photo", w, 24, w)[:, :, 0]).tobytes()
        for sched in (pes.schedule(24, "rows"), pes.schedule(24, [5, 2]), [24]):
            stream(pngb200, ctx, px, w, 24, fields, False, 4, 1000, sched, orc)


def test_rows_from_device_memory(pngb200, ctx, orc):
    import torch
    fields, w, h = dict(color=6, depth=8), 300, 90
    px = corpus.make("photo", w, h, 5).tobytes()
    for interlaced in (False, True):
        host = stream(pngb200, ctx, px, w, h, fields, interlaced, 6, 4096, pes.schedule(h, [7, 0, 13]))
        dev = torch.frombuffer(bytearray(px), dtype=torch.uint8).cuda()
        e = pngb200.PngEncoder(ctx, w, h, interlaced=interlaced, level=6, idat_chunk=4096, **fields)
        got, at = [], 0
        for n in pes.schedule(h, [7, 0, 13]):
            a, b = at * w * 4, (at + n) * w * 4
            e.push((dev.data_ptr() + a, b - a), pngb200.MEM_DEVICE)
            got.append(e.pop_all())
            at += n
        assert got == host, interlaced
        e.close()


def mixed(pngb200, ctx, count, seed):
    """count encoders of mixed formats, levels, interlacing and chunk sizes, with their storage and push schedule"""
    r = random.Random(seed)
    out = []
    for i in range(count):
        fields, w, h = FORMATS[i % len(FORMATS)]
        w, h = w + r.randint(0, 40), h + r.randint(0, 30)
        storage = noise(fields, w, h, seed * 1000 + i)
        kw = dict(interlaced=r.random() < 0.4, level=r.choice([0, 2, 4, 6, 8]), idat_chunk=r.choice([16, 700, 0]))
        sched = pes.schedule(h, [r.randint(0, 6) for _ in range(3)] + [1])
        out.append((fields, w, h, storage, kw, sched))
    return out


def test_batch_equals_pushes_made_alone(pngb200, ctx):
    cases = mixed(pngb200, ctx, 72, 3)
    alone = [pngb200.PngEncoder(ctx, w, h, **kw, **f) for f, w, h, _, kw, _ in cases]
    batch = [pngb200.PngEncoder(ctx, w, h, **kw, **f) for f, w, h, _, kw, _ in cases]
    pushes = [bands(s, h, sched) for _, _, h, s, _, sched in cases]
    rounds = max(len(p) for p in pushes)
    for k in range(rounds):
        items = [(batch[i], pushes[i][k]) for i in range(len(cases)) if k < len(pushes[i])]
        st = pngb200.png_encoder_push_batch(ctx, items)
        assert st == [0] * len(items)
        for i in range(len(cases)):
            if k < len(pushes[i]):
                alone[i].push(pushes[i][k])
                assert batch[i].pop_all() == alone[i].pop_all(), (i, k)
                assert batch[i].progress()[:5] == alone[i].progress()[:5], (i, k)
    for e in alone + batch:
        e.close()


def launch_deltas(pngb200, ctx, n):
    """kernel launches of each batch call that pushes one band into each of n encoders"""
    fields, w, h = dict(color=6, depth=8), 120, 40
    encs = [pngb200.PngEncoder(ctx, w, h, level=4, idat_chunk=512, **fields) for _ in range(n)]
    px = noise(fields, w, h, 9)
    deltas = []
    for rows in bands(px, h, pes.schedule(h, 8)):
        before = ctx.launches
        assert pngb200.png_encoder_push_batch(ctx, [(e, rows) for e in encs]) == [0] * n
        deltas.append(ctx.launches - before)
    for e in encs:
        e.close()
    return deltas


def test_launches_within_the_bound_whatever_the_count(pngb200, ctx):
    one, many = launch_deltas(pngb200, ctx, 1), launch_deltas(pngb200, ctx, 64)
    assert one == many and max(many) <= MAX_LAUNCHES and many[-1] == MAX_LAUNCHES, (one, many)


def test_batch_rejections_touch_nothing(pngb200, ctx):
    fields, w, h = dict(color=2, depth=8), 30, 20
    px = noise(fields, w, h, 4)
    a = pngb200.PngEncoder(ctx, w, h, level=4, **fields)
    b = pngb200.PngEncoder(ctx, w, h, level=4, **fields)
    a.push(px[: 3 * w * 3])
    other = pngb200.Context(0)
    c = pngb200.PngEncoder(other, w, h, **fields)
    try:
        before = (a.progress(), b.progress())
        lib = ctx._lib
        for items in ([(a, px[:w * 3]), (a, px[:w * 3])], [(a, px[:w * 3]), (c, px[:w * 3])]):
            with pytest.raises(pngb200.PNGB200Error):
                pngb200.png_encoder_push_batch(ctx, items)
        descs = (pngb200.PngEncoderPushDesc * 2)()
        descs[0].encoder, descs[0].rows, descs[0].n = a.handle, None, 5
        descs[1].encoder = b.handle
        assert lib.pngb200_png_encoder_push_batch(ctx.handle, descs, 2) == pngb200.ERR_BAD_ARGUMENT
        descs[0].rows, descs[0].n, descs[0].memspace = C.cast(C.c_char_p(px), C.c_void_p), w * 3, 7
        assert lib.pngb200_png_encoder_push_batch(ctx.handle, descs, 2) == pngb200.ERR_BAD_ARGUMENT
        assert descs[0].status == descs[1].status == 0
        assert (a.progress(), b.progress()) == before
        # item-level: not whole rows, past the height; the other item goes through
        assert pngb200.png_encoder_push_batch(ctx, [(a, px[:w * 3 - 1]), (b, px[:w * 3])]) == [pngb200.ERR_BAD_ARGUMENT, 0]
        assert pngb200.png_encoder_push_batch(ctx, [(a, px)]) == [pngb200.ERR_BAD_ARGUMENT]
        assert a.progress() == before[0]
        a.push(px[3 * w * 3:])
        assert a.progress()[4] == 1
        assert pngb200.png_encoder_push_batch(ctx, [(a, b"")]) == [pngb200.ERR_BAD_ARGUMENT]
        # a pending decode batch: the call is refused and no item moves
        from oracle import oracle
        img = bytes(np.random.default_rng(1).integers(0, 256, 64 * 64 * 4, dtype=np.uint8))
        zs = zlib.compress(oracle.png_filter(img, 64, 64, 32, 8), 6)
        dd = (pngb200.ImageDesc * 1)()
        out = C.create_string_buffer(len(img))
        dd[0].idat, dd[0].idat_len = C.cast(C.c_char_p(zs), C.c_void_p), len(zs)
        dd[0].width, dd[0].height, dd[0].volume, dd[0].depth = 64, 64, 32, 8
        dd[0].pixels, dd[0].pixels_cap = C.addressof(out), len(img)
        b.pop_all()
        before = b.progress()
        assert ctx._lib.pngb200_decode_batch_enqueue(ctx.handle, dd, 1, pngb200.MEM_HOST) == 0
        try:
            descs = (pngb200.PngEncoderPushDesc * 1)()
            descs[0].encoder, descs[0].rows, descs[0].n = b.handle, C.cast(C.c_char_p(px), C.c_void_p), w * 3
            assert lib.pngb200_png_encoder_push_batch(ctx.handle, descs, 1) == pngb200.ERR_BAD_ARGUMENT
            assert descs[0].status == 0 and b.progress() == before and b.pop_all() == []
        finally:
            assert ctx._lib.pngb200_decode_batch_finish(ctx.handle, dd, 1) == 0
        assert dd[0].status == 0 and out.raw == img
        assert pngb200.png_encoder_push_batch(ctx, [(b, px[w * 3: 2 * w * 3])]) == [0]
    finally:   # the handles go before their context
        for e in (a, b, c):
            e.close()
        other.close()


def test_create_refuses_images_a_push_could_not_finish(pngb200, ctx):
    """One push completes at most 1 GiB of filtered scanlines: an Adam7 image whose filtered stream is over that (its
    last row completes passes 1 to 6 at once) and a non-interlaced image with a scanline over it are refused when the
    handle is made, before any row is taken; the images just under the limit are accepted"""
    gib = 1 << 30
    with pytest.raises(pngb200.PNGB200Error) as e:
        pngb200.PngEncoder(ctx, 20000, 15000, color=6, depth=8, interlaced=True)
    assert e.value.status == pngb200.ERR_BAD_ARGUMENT
    with pytest.raises(pngb200.PNGB200Error) as e:
        pngb200.PngEncoder(ctx, gib // 4, 2, color=6, depth=8)           # pitch + 1 = 2^30 + 1
    assert e.value.status == pngb200.ERR_BAD_ARGUMENT
    ok = pngb200.PngEncoder(ctx, gib // 4 - 1, 2, color=6, depth=8)      # pitch + 1 = 2^30 - 3: one scanline a push
    ok.close()
    ok = pngb200.PngEncoder(ctx, 20000, 15000, color=6, depth=8)         # 1.2 GB of rows, pushed in bands
    ok.close()
    assert pngb200.filtered_size(16000, 16000, 32, True) <= gib
    ok = pngb200.PngEncoder(ctx, 16000, 16000, color=6, depth=8, interlaced=True)   # holds its storage: 1 GB
    ok.close()


def test_wide_image_in_bands_keeps_memory_flat(pngb200, ctx):
    fields, w, h = dict(color=6, depth=8), 7680, 480
    px = corpus.make("photo", w, h, 12).tobytes()
    e = pngb200.PngEncoder(ctx, w, h, level=2, **fields)
    pieces, held = [], []
    for rows in bands(px, h, pes.schedule(h, 16)):
        e.push(rows)
        pieces += e.pop_all()
        held.append(e.progress()[5])
    assert max(held) < 2 * held[0] and held[-1] < len(px) // 4, held
    (im,) = pngb200.png_decode_batch(ctx, [b"".join(pieces)])
    assert im.status == 0 and im.storage == px
    e.close()
