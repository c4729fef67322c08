"""The encoder edge corpus (tests/encode_corpus.py) at full size through the GPU encode path against the oracle: every
level, window exponent and wrapper set per stream in one batch, more streams than the launch has warp slots, a block at
the DF_GRAPH_CAP vertex cap, output capacity and the deflate bound, the streaming Deflator, and the filter / encode
stages on sub-byte, Adam7 and 16-bit images.  Needs an H100."""
from __future__ import annotations

import ctypes as C
import zlib

import numpy as np
import pytest

import corpus
import encode_corpus as ec
import test_emu_filter as ef

pytestmark = pytest.mark.gpu

LEVELS = [-1, 0, 1, 2, 3, 4, 5, 7, 8, 9, 11, 12, 13, 14]
FMTS = (ec.ZLIB, ec.GZIP, ec.IOS)


def bound(n: int) -> int:
    """pngb200_deflate_bound, csrc/pngb200_api.cu: `return n + n / 2 + 4096;`"""
    return n + n // 2 + 4096


def gpu_cases(level):
    cases = [c for fam in ec.FAMILIES for c in ec.build(fam, "gpu")]
    if level >= 11:     # keep the oracle's unlimited-attempt levels to a few seconds
        cases = [c for c in cases if c.family != "png"]
    return cases


def exponent_of(case, i):
    return int(case.name[1:case.name.index("p")]) if case.family == "window" else (8, 9, 12, 15)[i % 4]


@pytest.mark.parametrize("level", LEVELS)
def test_corpus_with_per_stream_formats_and_exponents(pngb200, ctx, orc, level):
    """one batch per level; wrapper and window exponent differ from stream to stream; every case reaches its edge"""
    cases = gpu_cases(level)
    fmts = [FMTS[i % 3] for i in range(len(cases))]
    exps = [exponent_of(c, i) for i, c in enumerate(cases)]
    got = pngb200.deflate_batch(ctx, [c.data for c in cases], level, fmts, exps)
    for c, fmt, e, (st, out) in zip(cases, fmts, exps, got):
        want = orc.deflate(c.data, level, fmt, e)
        assert st == 0 and out == want, (c.name, level, fmt, e)
        assert len(out) <= bound(len(c.data))
        if level in (0, 4, 9, 13):
            ec.check_reach(c, want, fmt, level, e)


def test_more_streams_than_warp_slots(pngb200, ctx, orc):
    """run_deflate launches min(count, budget / stride, 8 x SMs) warp slots: 1300 small streams outnumber 8 x 132, and a
    4 MiB level-8 stream in the second batch makes each slot's graph 2^21 vertices, so only a few dozen slots fit the
    budget; every slot serves stream after stream with other levels, wrappers and exponents"""
    tiny = ec.build("tiny", "gpu") + ec.build("lazy", "gpu") + [c for c in ec.build("window", "gpu") if c.name.startswith("e8")]
    streams = [tiny[i % len(tiny)].data for i in range(1300)]
    levels = [LEVELS[(i * 7) % len(LEVELS)] for i in range(1300)]
    fmts = [FMTS[i % 3] for i in range(1300)]
    exps = [(8, 15, 9, 12)[(i // 3) % 4] for i in range(1300)]
    got = pngb200.deflate_batch(ctx, streams, levels, fmts, exps)
    for d, lv, f, e, (st, out) in zip(streams, levels, fmts, exps, got):
        assert st == 0 and out == orc.deflate(d, lv, f, e), (len(d), lv, f, e)
    big = corpus.make("photo", 1024, 1024, 9).tobytes()
    streams = [big] + streams[:300]
    got = pngb200.deflate_batch(ctx, streams, [8] + levels[:300], [ec.ZLIB] + fmts[:300], [15] + exps[:300])
    assert got[0][0] == 0 and got[0][1] == orc.deflate(big, 8)
    for d, lv, f, e, (st, out) in zip(streams[1:], levels, fmts, exps, got[1:]):
        assert st == 0 and out == orc.deflate(d, lv, f, e), (len(d), lv, f, e)


def block_ends(orc, stream):
    """output offset at which each block of a zlib stream ends (the oracle's block trace)"""
    L = orc.lib()
    L.orc_debug_block_starts.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_size_t]
    L.orc_debug_block_starts.restype = C.c_size_t
    cap = 1 << 12
    trace = (C.c_uint64 * (3 * cap))()
    n = L.orc_debug_block_starts(orc.ZLIB, stream, len(stream), trace, cap)
    return [trace[3 * i + 1] for i in range(1, n)]


def test_block_at_the_graph_cap(pngb200, ctx, orc):
    """a 6.5 MB level-8 stream: full-mode blocks grow 2047, 4095 ... up to DF_GRAPH_CAP - 1 vertices, then stay there"""
    img = corpus.make("photo", 1600, 1024, 12).reshape(1024, -1)
    data = corpus.filter_rows_numpy(img, 4)
    (st, out), = pngb200.deflate_batch(ctx, [data], 8)
    want = orc.deflate(data, 8)
    assert st == 0 and out == want
    sizes = ec.full_blocks(len(data))
    assert sizes[-3] == sizes[-2] == ec.DF_GRAPH_CAP - 1 > sizes[-4]
    assert block_ends(orc, want) == list(np.cumsum(sizes)[:-1])
    assert zlib.decompress(out) == data


def raw_deflate(pngb200, ctx, data, level, fmt, caps):
    n = len(caps)
    descs = (pngb200.DeflateDesc * n)()
    src = C.create_string_buffer(data, len(data))
    dsts = [C.create_string_buffer(max(cap, 1)) for cap in caps]
    for i, cap in enumerate(caps):
        descs[i].src, descs[i].src_len = C.addressof(src), len(data)
        descs[i].dst, descs[i].dst_cap = C.addressof(dsts[i]), cap
        descs[i].format, descs[i].level, descs[i].exponent = fmt, level, 15
    ctx.check(ctx._lib.pngb200_deflate_batch(ctx.handle, descs, n, pngb200.MEM_HOST))
    return [(descs[i].status, dsts[i].raw[:descs[i].produced] if descs[i].status == 0 else None) for i in range(n)]


@pytest.mark.parametrize("level", [0, 4, 9])
def test_output_capacity_and_bound(pngb200, ctx, orc, level):
    """dst_cap 0, 1 and len - 1 fail with ERR_OUTPUT_CAPACITY, len succeeds; noise (the least compressible input) stays
    inside pngb200_deflate_bound"""
    data = ec.build("png", "gpu")[0].data
    for fmt in FMTS:
        want = orc.deflate(data, level, fmt)
        got = raw_deflate(pngb200, ctx, data, level, fmt, [0, 1, len(want) - 1, len(want)])
        assert [st for st, _ in got] == [pngb200.ERR_OUTPUT_CAPACITY] * 3 + [0]
        assert got[3][1] == want
    noise = np.random.default_rng(8).integers(0, 256, 300000, dtype=np.uint8).tobytes()
    (st, out), = pngb200.deflate_batch(ctx, [noise], level, ec.GZIP)
    assert st == 0 and out == orc.deflate(noise, level, ec.GZIP) and len(out) <= bound(len(noise))


@pytest.mark.parametrize("fmt,exponent", [(ec.ZLIB, 15), (ec.GZIP, 15), (ec.ZLIB, 8)])
def test_streaming_deflator_push_sizes(pngb200, ctx, orc, fmt, exponent):
    """pushes of 1 byte, of chunk_bytes - 1 and + 1, and empty non-final pushes; pop() hands out complete blocks only
    (none before the last push), pull() the rest; the concatenation is the one-shot stream"""
    chunk = 1000
    data = ec.build("png", "gpu")[1].data[:20000]
    z = pngb200.Deflator(ctx, fmt, level=9, exponent=exponent, chunk_bytes=chunk)
    at, parts = 0, []
    for size in [1, chunk - 1, 0, chunk + 1, 1, 0] * 8:
        z.push(data[at:at + size])
        at += size
        assert z.pop() is None
    z.push(data[at:], last=True)
    while (b := z.pop()) is not None:
        assert len(b) == chunk
        parts.append(b)
    while (b := z.pull()) is not None:
        parts.append(b)
    z.close()
    want = orc.deflate(data, 9, fmt, exponent)
    assert b"".join(parts) == want
    assert all(len(p) == chunk for p in parts[:-1]) and 0 < len(parts[-1]) <= chunk


def filter_images():
    rng = np.random.default_rng(30)
    images = [ef.image(rng, w, h, vol, vol, il) for vol in (1, 2, 4) for w in range(1, 18) for h, il in ((3, False), (6, True))]
    images += [ef.image(rng, w, h, 24, 8, True) for w in range(1, 10) for h in range(1, 10)]
    images += [ef.image(rng, w, h, vol, 16, il) for vol in (32, 64) for (w, h) in ((13, 7), (40, 11)) for il in (False, True)]
    images += [(bytes(40 * 9 * 4), 40, 9, 32, 8, False), (b"\x80" * 33 * 5, 33, 5, 8, 8, False)]
    for first, second in ((0, 1), (1, 2), (2, 3), (3, 4)):
        images.append((ef.tie_rows(rng, first, second), 6, 2, 8, 8, False))
    return images


def test_filter_edges(pngb200, ctx, orc):
    """the emulator's filter cases in one filter_batch: ties, sub-byte widths 1..17, Adam7 1x1..9x9, 16-bit samples"""
    images = filter_images()
    got = pngb200.filter_batch(ctx, [dict(pixels=st, width=w, height=h, volume=v, depth=d, interlaced=il)
                                     for st, w, h, v, d, il in images])
    for (st, w, h, v, d, il), f in zip(images, got):
        assert f == orc.png_filter(st, w, h, v, d, il), (w, h, v, d, il)


@pytest.mark.parametrize("level", [0, 4, 9])
def test_encode_sub_byte_and_adam7(pngb200, ctx, orc, level):
    """encode_batch (filter + deflate) on the same images == oracle.deflate(oracle.png_filter(...), level)"""
    images = filter_images()
    got = pngb200.encode_batch(ctx, [dict(pixels=st, width=w, height=h, volume=v, depth=d, interlaced=il)
                                     for st, w, h, v, d, il in images], level=level)
    for (st, w, h, v, d, il), (status, idat) in zip(images, got):
        assert status == 0 and idat == orc.deflate(orc.png_filter(st, w, h, v, d, il), level), (w, h, v, d, il)
