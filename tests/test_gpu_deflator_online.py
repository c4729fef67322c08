"""The online deflator (pngb200_deflator_create_online, pngb200_deflator_push_batch) on the GPU: after every push,
pop() and pull() return exactly what the streaming restatement of LZ77.Deflator (tests/deflate_stream.c) returns;
the committed level-9 outputs come out in PNG.Encoder's call order; a long level-8 stream keeps its device state
bounded; a batch push is the same pushes made alone, refuses bad calls whole, and makes at most one launch."""
from __future__ import annotations

import ctypes
import os
import random
import zlib

import pytest

import deflate_stream as ds
import pngio
from conftest import GOLDEN

pytestmark = pytest.mark.gpu



def text(n, seed):
    r = random.Random(seed)
    words = [bytes(r.choice(b"abcdefghijklmnop") for _ in range(r.randint(2, 9))) for _ in range(400)]
    out = bytearray()
    while len(out) < n:
        out += r.choice(words) + b" "
        if r.random() < 0.02:
            out += bytes(r.getrandbits(8) for _ in range(r.randint(1, 60)))
        if r.random() < 0.005:
            out += bytes([r.getrandbits(8)]) * r.randint(100, 700)
    return bytes(out[:n])


def take(d, final):
    """pop() until nil, then pull() (until nil after the last push, once before it)"""
    out = []
    while (c := d.pop()) is not None:
        out.append(c)
    while (c := d.pull()) is not None:
        out.append(c)
        if not final:
            break
    return out


def replay(pngb200, ctx, data, fmt, level, exponent, sizes, chunk):
    g = pngb200.Deflator(ctx, fmt, level, exponent, chunk_bytes=chunk, online=True)
    o = ds.StreamingDeflator(fmt, level, exponent, chunk)
    pieces = ds.cuts(len(data), sizes)
    for k, (a, b) in enumerate(pieces + [(0, 0)]):
        last = k == len(pieces)
        g.push(data[a:b], last=last)
        o.push(data[a:b], last)
        assert take(g, last) == take(o, last), (level, fmt, k)
    assert g.pop() is None and g.pull() is None
    return g


@pytest.mark.parametrize("level", [0, 3, 4, 7, 8, 9, 13])
def test_every_push_hands_out_what_the_reference_does(pngb200, ctx, level):
    n = 20000 if level == 13 else 400000 if level >= 8 else 1500000
    data = text(n, level)
    for fmt, exponent, sizes, chunk in ((ds.ZLIB, 15, [65544], 65544), (ds.GZIP, 8, [4097, 1, 258, 259, 70001], 4000),
                                        (ds.IOS, 8, [1, 4096, 7, 12345], 1000)):
        replay(pngb200, ctx, data, fmt, level, exponent, sizes, chunk).close()


def test_tiny_and_empty_streams(pngb200, ctx):
    for fmt in (ds.ZLIB, ds.GZIP, ds.IOS):
        for pushes in ([b"a", b"b"], [b"", b"ab", b""], [b"x"], [], [b"abc"]):
            replay(pngb200, ctx, b"".join(pushes), fmt, 9, 15, [1], 65544).close()


@pytest.mark.parametrize("name", sorted(f for f in os.listdir(os.path.join(GOLDEN, "encode")) if f.startswith("out-")))
def test_golden_outputs_in_png_encoder_call_order(pngb200, ctx, name):
    """one filtered row per push, pop() after each, then push([], last: true) and pull() until nil: the committed
    file's IDAT chunks, the first of them before the last push"""
    raw = open(os.path.join(GOLDEN, "encode", name), "rb").read()
    png = pngio.parse(raw)
    filtered = zlib.decompress(png.idat)
    pitch = len(filtered) // png.height
    z = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, level=9, online=True)
    chunks, early = [], 0
    for y in range(png.height):
        z.push(filtered[y * pitch:(y + 1) * pitch])
        while (b := z.pop()) is not None:
            chunks.append(b)
    early = len(chunks)
    z.push(b"", last=True)
    while (b := z.pull()) is not None:
        chunks.append(b)
    assert b"".join(chunks) == png.idat
    assert [len(c) for c in chunks] == [len(c) for c in pngio.idat_chunks(raw)]
    assert early > 0 or len(chunks) == 1
    z.close()


def test_long_level8_stream_is_bounded(pngb200, ctx, orc):
    """6 MB at level 8: the doubling blocks reach 2^21 - 1 vertices.  Every byte is dequeued once, at most 259 bytes
    stay pending after a push that compresses, and the device state stays within the dictionary, the graph of the
    largest block, the live input and the output of one launch (peak about 360 MB of device memory)"""
    data = text(6 << 20, 77)
    g = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, level=8, online=True)
    out, peak = [], 0
    total = 0
    for a, b in ds.cuts(len(data), [65544]):
        g.push(data[a:b])
        total += b - a
        dequeued, written, blocks, held = g.stats()
        assert dequeued <= total
        if total - dequeued > 4096 or dequeued:
            assert total - dequeued <= 4096 + 65544
        peak = max(peak, held)
        out += take(g, False)
    before = g.stats()
    g.push(b"", last=True)
    out += take(g, True)
    assert b"".join(out) == orc.deflate(data, 8)
    dequeued, written, blocks, held = g.stats()
    assert dequeued == len(data) and written == len(b"".join(out)) and blocks > before[2] >= 11
    # dictionary, graph (128 B per vertex + upstream words), live input (block + window), one launch's output
    live = (1 << 21) + 2 * 32768 + 65544 + 4096 + 16
    bound = (64 << 10) + 1.25 * ((512 << 10) + 132 * ((1 << 21) + 3) + live + 1.5 * (live + (1 << 21)) + 8192)
    assert peak <= bound, (peak, bound)
    g.close()


def test_dequeued_after_every_push_is_the_references(pngb200, ctx):
    """the 4096 guard, the 258 / 259 lookahead and the skip run of a long match, seen through stats()"""
    data = text(300000, 3)
    for level in (2, 5, 9):
        g = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, level=level, online=True)
        o = ds.StreamingDeflator(ds.ZLIB, level, 15, ds.CHUNK)
        for a, b in ds.cuts(len(data), [5000, 9000, 1, 4096]):
            g.push(data[a:b])
            o.push(data[a:b])
            dequeued, written, blocks, pending = o.progress()
            assert g.stats()[:3] == (dequeued, written, blocks), (level, a)
        g.close()


def test_batch_equals_pushes_made_alone(pngb200, ctx):
    specs = [(pngb200.FORMAT_ZLIB, 9, 15), (pngb200.FORMAT_GZIP, 4, 8), (pngb200.FORMAT_IOS, 1, 15),
             (pngb200.FORMAT_ZLIB, 13, 10), (pngb200.FORMAT_ZLIB, 0, 8), (pngb200.FORMAT_GZIP, 8, 15)]
    data = [text(120000 if s[1] != 13 else 30000, i) for i, s in enumerate(specs)]
    rng = random.Random(4)
    batched = [pngb200.Deflator(ctx, *s, online=True) for s in specs]
    alone = [pngb200.Deflator(ctx, *s, online=True) for s in specs]
    at = [0] * len(specs)
    outs_b = [[] for _ in specs]
    outs_a = [[] for _ in specs]
    while any(a <= len(d) for a, d in zip(at, data)):
        items = []
        for i, d in enumerate(data):
            if at[i] > len(d) or rng.random() < 0.2:
                continue
            step = rng.choice([1, 700, 4097, 30000])
            piece, last = d[at[i]:at[i] + step], at[i] + step >= len(d) and rng.random() < 0.5
            at[i] = at[i] + step if not last else len(d) + 1
            if at[i] >= len(d) and not last:
                at[i] = len(d)
            items.append((i, piece, last))
        st = pngb200.deflator_push_batch(ctx, [(batched[i], p, last) for i, p, last in items])
        assert st == [0] * len(items)
        for i, p, last in items:
            alone[i].push(p, last=last)
            outs_b[i] += take(batched[i], last)
            outs_a[i] += take(alone[i], last)
            assert outs_b[i] == outs_a[i]
            assert batched[i].stats()[:3] == alone[i].stats()[:3]
    for i, s in enumerate(specs):
        assert b"".join(outs_b[i]) == ds_oracle(data[i], *s)
    for z in batched + alone:
        z.close()


def ds_oracle(data, fmt, level, exponent):
    d = ds.StreamingDeflator(fmt, level, exponent, ds.CHUNK)
    d.push(data, True)
    return b"".join(ds.drain(d, True))


def test_batch_rejections_touch_nothing(pngb200, ctx):
    a = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, 4, online=True)
    b = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, 4, online=True)
    buffered = pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, 4)
    other_ctx = pngb200.Context(0)
    other = pngb200.Deflator(other_ctx, pngb200.FORMAT_ZLIB, 4, online=True)
    data = text(10000, 1)
    L = ctx._lib
    for bad in ([(a, data, False), (a, data, False)], [(a, data, False), (buffered, data, False)],
                [(a, data, False), (other, data, False)]):
        with pytest.raises(pngb200.PNGB200Error) as e:
            pngb200.deflator_push_batch(ctx, bad)
        assert e.value.status == pngb200.ERR_BAD_ARGUMENT
    descs = (pngb200.DeflatorPushDesc * 2)()
    descs[0].deflator, descs[0].data, descs[0].n = a.handle, None, 0
    descs[1].deflator, descs[1].data, descs[1].n = b.handle, None, 5
    assert L.pngb200_deflator_push_batch(ctx.handle, descs, 2) == pngb200.ERR_BAD_ARGUMENT
    descs[1].deflator, descs[1].n = None, 0
    assert L.pngb200_deflator_push_batch(ctx.handle, descs, 2) == pngb200.ERR_BAD_ARGUMENT
    assert L.pngb200_deflator_push_batch(None, descs, 1) == pngb200.ERR_BAD_ARGUMENT
    assert L.pngb200_deflator_push_batch(ctx.handle, None, 1) == pngb200.ERR_BAD_ARGUMENT
    assert L.pngb200_deflator_stats(buffered.handle, (ctypes.c_uint64 * 4)()) == pngb200.ERR_BAD_ARGUMENT
    assert a.stats()[:3] == b.stats()[:3] == (0, 2, 0)
    # nothing was touched: both still compress the stream from its start
    a.push(data, last=True)
    assert b"".join(take(a, True)) == ds_oracle(data, pngb200.FORMAT_ZLIB, 4, 15)
    with pytest.raises(pngb200.PNGB200Error):
        a.push(b"x")
    for z in (a, b, buffered, other):
        z.close()
    other_ctx.close()


@pytest.mark.parametrize("n", [1, 64])
def test_one_launch_per_batch(pngb200, ctx, n):
    levels = [[0, 1, 4, 7, 9][i % 5] for i in range(n)]
    zs = [pngb200.Deflator(ctx, pngb200.FORMAT_ZLIB, level=lv, online=True) for lv in levels]
    data = [text(140000, i) for i in range(n)]
    for k, (a, b) in enumerate(ds.cuts(140000, [65544])):
        before = ctx.launches
        st = pngb200.deflator_push_batch(ctx, [(z, d[a:b], False) for z, d in zip(zs, data)])
        assert st == [0] * n and ctx.launches - before <= 1
    before = ctx.launches
    pngb200.deflator_push_batch(ctx, [(z, b"", True) for z in zs])
    assert ctx.launches - before == 1
    for z, d, lv in zip(zs, data, levels):
        assert b"".join(take(z, True)) == ds_oracle(d, pngb200.FORMAT_ZLIB, lv, 15)
        z.close()
