"""The whole-stream wave engines forced one at a time on the GPU: inflate mode 3 (inflate_wave_kernel), 4 (the round-1
inflate_parallel_kernel / inflate_parallel_kernel3) and 6 (inflate_cells_kernel), with no segments and no split.  Every
stream is at least 8 KiB compressed, so none of them goes to the serial kernel instead.  Status, error payload, bytes
and checksum are compared with the oracle and zlib, including the streams that fall back to the serial decoder."""
import gzip
import zlib

import pytest

import corpus

pytestmark = pytest.mark.gpu

ENGINES = {3: "inflate_wave_kernel", 4: "inflate_parallel_kernel", 6: "inflate_cells_kernel"}
MIN_COMPRESSED = 8 << 10   # parallel_threshold: smaller streams are decoded by the serial kernel


def _inflate(pngb200, ctx, mode, streams, fmts, caps):
    ctx.set_inflate_mode(mode)
    try:
        got = pngb200.inflate_batch(ctx, streams, fmts, caps=caps)
        engine = ctx.last_inflate_engine()
    finally:
        ctx.set_inflate_mode(0)
    return got, engine


def _check(orc, got, streams, fmts, caps):
    for k, ((st, out, d), s, f, cap) in enumerate(zip(got, streams, fmts, caps)):
        ost, oout, ores = orc.inflate(s, f, cap)
        assert st == ost, (k, st, ost)
        assert (d.err_a, d.err_b) == (ores.a, ores.b), k
        if ost == 0:
            assert out == oout, k
            assert d.checksum == ores.checksum, k


def _images():
    """filtered scanlines of the synthetic corpora"""
    out = []
    for i, (kind, w, h, wide) in enumerate([("photo", 640, 480, False), ("graphic", 1600, 1200, False),
                                            ("noise", 256, 192, False), ("photo", 512, 300, True)]):
        im = corpus.make(kind, w, h, 70 + i, wide)
        out.append(corpus.zlib_png_stream(im, 8 if wide else 4, 1)[0])
    return out


@pytest.mark.parametrize("mode", sorted(ENGINES))
def test_engine_matches_oracle_and_zlib(pngb200, ctx, orc, mode):
    """zlib levels 1/6/9 and the reference encoder's level-4 and level-9 streams of the corpora as zlib, the same data as
    gzip and raw streams: bytes, Adler-32 / CRC-32 and status against the oracle and zlib"""
    streams, fmts = [], []
    for f in _images():
        for level in (1, 6, 9):
            streams.append(zlib.compress(f, level))
            fmts.append(pngb200.FORMAT_ZLIB)
        for level in (4, 9):
            streams.append(orc.deflate(f, level))
            fmts.append(pngb200.FORMAT_ZLIB)
        streams.append(gzip.compress(f, 6, mtime=0))
        fmts.append(pngb200.FORMAT_GZIP)
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        streams.append(c.compress(f) + c.flush())
        fmts.append(pngb200.FORMAT_IOS)
    assert min(len(s) for s in streams) >= MIN_COMPRESSED
    plain = [zlib.decompress(s, 47 if f == pngb200.FORMAT_GZIP else -15 if f == pngb200.FORMAT_IOS else 15)
             for s, f in zip(streams, fmts)]
    caps = [len(p) for p in plain]
    got, engine = _inflate(pngb200, ctx, mode, streams, fmts, caps)
    assert engine == ENGINES[mode]
    for k, ((st, out, d), p) in enumerate(zip(got, plain)):
        assert st == 0 and out == p, k
    _check(orc, got, streams, fmts, caps)


@pytest.mark.parametrize("mode", sorted(ENGINES))
def test_engine_errors_take_the_serial_fallback(pngb200, ctx, orc, mode):
    """a truncated stream, a bad Adler-32 trailer and a stream damaged in a late block: the engine hands them to the
    serial decoder or compares the trailer itself; statuses and error payloads are the oracle's"""
    f = _images()[0]
    z = zlib.compress(f, 6)
    bad_adler = bytearray(z)
    bad_adler[-1] ^= 0x5a
    late = bytearray(z)
    for at in range(len(z) * 7 // 8, len(z) * 7 // 8 + 64, 4):
        late[at] ^= 0xff
    streams = [z[: len(z) * 2 // 3], bytes(bad_adler), bytes(late), z]
    assert min(len(s) for s in streams) >= MIN_COMPRESSED
    fmts = [pngb200.FORMAT_ZLIB] * len(streams)
    caps = [len(f)] * len(streams)
    got, engine = _inflate(pngb200, ctx, mode, streams, fmts, caps)
    assert engine == ENGINES[mode]
    assert [g[0] != 0 for g in got] == [True, True, True, False]
    assert got[1][0] == pngb200.ERR_STREAM_CHECKSUM
    assert got[3][1] == f
    _check(orc, got, streams, fmts, caps)


def test_round1_engine_with_more_streams_than_three_per_sm(pngb200, ctx, orc):
    """more than 3 x SMs streams in mode 4: the 64-register inflate_parallel_kernel runs (not kernel3)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms + 9
    streams, plain = [], []
    for i in range(n):
        f = corpus.zlib_png_stream(corpus.make("noise", 96, 64, 200 + i), 4, 1)[0]
        streams.append(zlib.compress(f, 1 + i % 9))
        plain.append(f)
    assert min(len(s) for s in streams) >= MIN_COMPRESSED
    fmts = [pngb200.FORMAT_ZLIB] * n
    caps = [len(p) for p in plain]
    got, engine = _inflate(pngb200, ctx, 4, streams, fmts, caps)
    assert engine == "inflate_parallel_kernel"
    for k, ((st, out, d), p) in enumerate(zip(got, plain)):
        assert st == 0 and out == p and d.checksum == zlib.adler32(p), k
    _check(orc, got, streams, fmts, caps)
