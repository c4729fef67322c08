"""The crafted DEFLATE corpus (tests/deflate_craft.py) at full size on the GPU: every inflate mode and engine, segments,
the split head + tail with its switch out of symbolic mode, gzip and raw wrappers and the streaming inflator, against
the oracle.  Valid streams must be decoded by the path under test itself: no serial fallback, no segment or split
fallback, so that a wrong symbolic decode cannot hide behind the whole-stream re-decode."""
from __future__ import annotations

import functools
import os
import zlib

import pytest

import deflate_craft as dc

pytestmark = pytest.mark.gpu

ENGINES = {3: "inflate_wave_kernel", 4: "inflate_parallel_kernel", 6: "inflate_cells_kernel"}
SIZES = {"far_window": 1_500_000, "sparse_trees": 1_500_000, "empty_blocks": 1_500_000, "fixed_long": 1_500_000,
         "rle_258": 5_000_000, "header_straddle": 1_200_000, "hdist32_unused": 1_200_000}
BAD_PREFIX = 200_000


@functools.lru_cache(maxsize=None)
def case(name, size=None, seed=5):
    return dc.build(name, size or SIZES.get(name, BAD_PREFIX), seed)


def check(orc, got, streams, fmts, caps):
    for k, ((st, out, d), s, f, cap) in enumerate(zip(got, streams, fmts, caps)):
        ost, oout, ores = orc.inflate(s, f, cap)
        assert (st, d.err_a, d.err_b) == (ost, ores.a, ores.b), k
        if ost == 0:
            assert out == oout, k
            assert (d.checksum, d.blocks) == (ores.checksum, ores.blocks), k


def inflate(pngb200, ctx, mode, streams, fmts, caps):
    ctx.set_inflate_mode(mode)
    try:
        got = pngb200.inflate_batch(ctx, streams, fmts, caps=caps)
        return got, ctx.last_inflate_engine(), ctx.inflate_stats(len(streams))
    finally:
        ctx.set_inflate_mode(0)


@pytest.mark.parametrize("mode", [1, 3, 4, 6, 0])
def test_inflate_modes(pngb200, ctx, orc, mode):
    """mode 1: serial kernel; 3 / 4 / 6: one engine forced; 0: the automatic choice"""
    valid = [case(n).stream("zlib") for n in sorted(dc.CASES)]
    streams, caps = [v[0] for v in valid], [len(v[1]) for v in valid]
    fmts = [pngb200.FORMAT_ZLIB] * len(streams)
    got, engine, stats = inflate(pngb200, ctx, mode, streams, fmts, caps)
    if mode in ENGINES:
        assert engine == ENGINES[mode]
        assert stats["fallbacks"] == 0
    elif mode == 1:
        assert engine == ""
    for (st, out, _), (_, plain, _) in zip(got, valid):
        assert st == 0 and out == plain
    check(orc, got, streams, [orc.ZLIB] * len(streams), caps)
    bad = [case(n).stream("zlib") for n in sorted(dc.INVALID)]
    streams, caps = [b[0] for b in bad], [len(b[1]) + 4096 for b in bad]
    got, engine, _ = inflate(pngb200, ctx, mode, streams, fmts[:1] * len(streams), caps)
    if mode in ENGINES:
        assert engine == ENGINES[mode]
    for (st, _, d), n in zip(got, sorted(dc.INVALID)):
        assert (st, d.err_a, d.err_b) == (case(n).status, *case(n).err), n
    check(orc, got, streams, [orc.ZLIB] * len(streams), caps)


def test_gzip_and_raw(pngb200, ctx, orc):
    streams, fmts, ofmts, plains = [], [], [], []
    for n in sorted(dc.CASES):
        for wrapper, f, of in (("gzip", pngb200.FORMAT_GZIP, orc.GZIP), ("raw", pngb200.FORMAT_IOS, orc.IOS)):
            z, plain, _ = case(n).stream(wrapper)
            streams.append(z), fmts.append(f), ofmts.append(of), plains.append(plain)
    caps = [len(p) for p in plains]
    got = pngb200.inflate_batch(ctx, streams, fmts, caps=caps)
    for (st, out, _), p in zip(got, plains):
        assert st == 0 and out == p
    check(orc, got, streams, ofmts, caps)


BIG = {"far_window": 2_200_000, "header_straddle": 1_200_000, "sparse_trees": 3_500_000, "empty_blocks": 1_300_000}


def big_streams():
    """families with split points at 1 MiB and more of compressed and of decoded bytes (the planners' minimum)"""
    out = [(n, case(n, BIG[n], seed=7)) for n in sorted(BIG)]
    out += [("far_window", case("far_window", BIG["far_window"], seed=8)),
            ("far_window", case("far_window", BIG["far_window"], seed=9))]
    for n, c in out:
        z, plain, _ = c.stream("zlib")
        assert min(len(z), len(plain)) >= 1 << 20, n
    return out


def test_segments_auto_mode_few_streams(pngb200, ctx, orc):
    big = big_streams()[:4]
    valid = [c.stream("zlib") for _, c in big]
    streams, caps = [v[0] for v in valid], [len(v[1]) for v in valid]
    got, _, stats = inflate(pngb200, ctx, 0, streams, [pngb200.FORMAT_ZLIB] * len(streams), caps)
    seg = ctx.segment_stats()
    assert seg["streams"] == len(streams) and seg["segments"] >= 4 * len(streams) and seg["fallbacks"] == 0, seg
    for (st, out, _), (_, plain, _) in zip(got, valid):
        assert st == 0 and out == plain
    check(orc, got, streams, [orc.ZLIB] * len(streams), caps)


# ---- split: a direct head and a symbolic tail per stream, on few CTA slots ----
SLOTS = 8   # 6 streams on 8 slots


def make_ctx(pngb200, **env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return pngb200.Context(0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def split_ctx(pngb200):
    c = make_ctx(pngb200, PNGB200_PLAN_SLOTS=str(SLOTS), PNGB200_SPLIT="1")
    yield c
    c.close()


def one_row_image(c: dc.Case):
    """the case's bytes as one scanline of an 8-bit grey image: a stored block holding filter byte 0 goes in front
    (it ends on a byte boundary, so the case's blocks follow unchanged)"""
    raw, plain, _ = c.stream("raw")
    data = b"\x00" + plain
    z = b"\x78\x9c" + bytes([0x00, 0x01, 0x00, 0xFE, 0xFF, 0x00]) + raw + zlib.adler32(data).to_bytes(4, "big")
    assert zlib.decompress(z) == data
    return dict(idat=z, width=len(plain), height=1, volume=8, depth=8), plain


def decode_device(pngb200, ctx, jobs):
    import torch
    descs = (pngb200.ImageDesc * len(jobs))()
    keep = []
    for i, j in enumerate(jobs):
        idat = torch.frombuffer(bytearray(j["idat"]), dtype=torch.uint8).cuda()
        size = pngb200.storage_size(j["width"], j["height"], j["volume"])
        pix = torch.full((size,), 0xA5, dtype=torch.uint8, device="cuda")
        keep.append((idat, pix))
        descs[i].idat, descs[i].idat_len = idat.data_ptr(), idat.numel()
        descs[i].pixels, descs[i].pixels_cap = pix.data_ptr(), size
        descs[i].width, descs[i].height = j["width"], j["height"]
        descs[i].volume, descs[i].depth = j["volume"], j["depth"]
        descs[i].interlaced, descs[i].format = 0, 0
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_decode_batch(ctx.handle, descs, len(jobs), pngb200.MEM_DEVICE))
    return [dict(status=descs[i].status, checksum=descs[i].checksum, blocks=descs[i].blocks,
                 pixels=keep[i][1].cpu().numpy().tobytes()) for i in range(len(jobs))]


def test_split_and_switch(pngb200, split_ctx, orc):
    big = big_streams()
    assert len(big) == 6
    imgs = [one_row_image(c) for _, c in big]
    got = decode_device(pngb200, split_ctx, [j for j, _ in imgs])
    seg = split_ctx.segment_stats()
    assert seg == dict(streams=6, segments=12, fallbacks=0), seg
    sp = split_ctx.split_stats()
    assert sp["tail_bytes"] > 0 and sp["switched"] >= 1, sp
    for g, (j, plain) in zip(got, imgs):
        _, _, ores = orc.inflate(j["idat"], orc.ZLIB, len(plain) + 1)
        assert g["status"] == 0 and g["pixels"] == plain
        assert (g["checksum"], g["blocks"]) == (ores.checksum, ores.blocks)


@pytest.mark.parametrize("name", ["empty_blocks", "header_straddle", "far_window"])
def test_streaming_inflator_pushes_cut_blocks(pngb200, ctx, name):
    """pushes that end inside stored-block headers, stored data and dynamic headers (a few bits past every tenth block
    start), then big pushes"""
    z, plain, blocks = case(name, 400_000).stream("zlib")
    cuts = sorted({b // 8 + d for b, _, _ in blocks[::10] for d in (0, 1, 3)} | {len(z) // 2, len(z) - 3})
    cuts = [c for c in cuts if 0 < c < len(z)] + [len(z)]
    inf = pngb200.Inflator(ctx, pngb200.FORMAT_ZLIB)
    try:
        out, at, status = b"", 0, None
        for c in cuts:
            if c <= at:
                continue
            status = inf.push(z[at:c])
            at = c
            out += inf.pull_all()
        assert status == pngb200.OK and out == plain
    finally:
        inf.close()
