"""The streaming restatement of LZ77.Deflator (tests/deflate_stream.c) on the CPU: for every push schedule its chunks
concatenate to orc_deflate's stream, the committed level-9 outputs come out chunk by chunk in PNG.Encoder's call order
with the first chunks before the last push, and the rules of DeflatorBuffers.push hold at their edges."""
from __future__ import annotations

import os
import random
import zlib

import pytest

import deflate_stream as ds
import pngio
from oracle import oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encode")
OUTPUTS = sorted(f for f in os.listdir(GOLDEN) if f.startswith("out-"))


def text(n, seed):
    r = random.Random(seed)
    words = [bytes(r.choice(b"abcdefghij") for _ in range(r.randint(2, 9))) for _ in range(80)]
    out = bytearray()
    while len(out) < n:
        out += r.choice(words) + b" "
        if r.random() < 0.01:
            out += bytes([r.getrandbits(8)]) * r.randint(100, 600)
    return bytes(out[:n])


def stream(data, fmt, level, exponent, sizes, chunk=ds.CHUNK):
    """(chunks after each push, the last push's included)"""
    d = ds.StreamingDeflator(fmt, level, exponent, chunk)
    got = []
    for a, b in ds.cuts(len(data), sizes):
        d.push(data[a:b])
        got.append(ds.drain(d))
    d.push(b"", True)
    got.append(ds.drain(d, True))
    assert d.pop() is None and d.pull() is None
    return got, d


@pytest.mark.parametrize("level", [0, 3, 4, 7, 8, 9, 13])
@pytest.mark.parametrize("sizes", [[1 << 20], [65544], [4097, 1, 258, 259], [1, 4096, 7], [333]])
def test_any_schedule_gives_the_one_shot_stream(level, sizes):
    data = text(12000 if level == 13 else 90000, level)
    for fmt, exponent in ((ds.ZLIB, 15), (ds.GZIP, 8), (ds.IOS, 8)):
        got, _ = stream(data, fmt, level, exponent, sizes, chunk=1000)
        flat = [c for push in got for c in push]
        assert b"".join(flat) == oracle.deflate(data, level, fmt, exponent)
        assert all(len(c) == 1000 for c in flat[:-1])


@pytest.mark.parametrize("name", OUTPUTS)
def test_golden_outputs_in_png_encoder_call_order(name):
    """one filtered row per push, pop() after each, then push([], last: true) and pull() until nil: the committed
    file's IDAT chunks, the first of them before the last push"""
    raw = open(os.path.join(GOLDEN, name), "rb").read()
    png = pngio.parse(raw)
    assert not png.interlaced
    filtered = zlib.decompress(png.idat)
    pitch = len(filtered) // png.height
    got, _ = stream(filtered, ds.ZLIB, 9, 15, [pitch])
    chunks = [c for push in got for c in push]
    assert b"".join(chunks) == png.idat
    assert [len(c) for c in chunks] == [len(c) for c in pngio.idat_chunks(raw)]
    if len(chunks) > 1:
        assert sum(len(p) for p in got[:-1]) > 0, "every chunk waited for the last push"


def progress_after(data, level, sizes, fmt=ds.ZLIB, exponent=15):
    d = ds.StreamingDeflator(fmt, level, exponent, 1)
    out = []
    for a, b in ds.cuts(len(data), sizes):
        d.push(data[a:b])
        out.append(d.progress())
    return out, d


def test_pending_4096_waits_and_4097_compresses():
    data = text(20000, 1)
    (p,), _ = progress_after(data[:4096], 4, [4096])
    assert p[0] == 0 and p[3] == 4096                 # DeflatorBuffers.swift:74: input.count > 4096 or last
    (p,), _ = progress_after(data[:4097], 4, [4097])
    assert p[0] > 0 and p[3] <= 259                   # lazy: no head is taken with 259 or fewer pending
    (p,), _ = progress_after(data[:4097], 3, [4097])
    assert p[3] <= 258                                # greedy and full: 258


def test_lookahead_is_tested_at_heads_only():
    """a match taken at the last head consumes its run past the lookahead point"""
    data = bytes(range(200)) + b"\x00" * 5000
    for level in (0, 4, 9):
        (p,), _ = progress_after(data, level, [len(data)])
        assert p[3] < 200


def test_block_filling_at_the_lookahead_is_written_by_a_later_push():
    """greedy on random bytes: literals only, a block every 2047.  The second block fills at position 4093; with 4355
    bytes pushed the next head (4094) sees exactly 258 pending, is not taken, and the full block waits for a later
    push that compresses; with 4356 it is written at once"""
    r = random.Random(5)
    data = bytes(r.getrandbits(8) for _ in range(12000))
    (p,), _ = progress_after(data[:4355], 0, [4355])
    assert p[2] == 1 and p[3] == 258
    (p,), _ = progress_after(data[:4356], 0, [4356])
    assert p[2] == 2
    ps, _ = progress_after(data[:4355 + 1 + 4097], 0, [4355, 1, 4097])
    assert [q[2] for q in ps] == [1, 1, 4]            # blocks fill at 2046, 4093, 6140 and 8187
    got, _ = stream(data, ds.ZLIB, 0, 15, [4355, 1, 4097], chunk=1)
    assert b"".join(c for push in got for c in push) == oracle.deflate(data, 0)


def test_tiny_streams_are_stored_whichever_pushes_bring_them():
    for fmt in (ds.ZLIB, ds.GZIP, ds.IOS):
        for pushes in ([b"a", b"b"], [b"", b"ab", b""], [b"x"], []):
            d = ds.StreamingDeflator(fmt, 9, 15, ds.CHUNK)
            for p in pushes:
                d.push(p)
            d.push(b"", True)
            data = b"".join(pushes)
            assert b"".join(ds.drain(d, True)) == oracle.deflate(data, 9, fmt, 15)


def test_gzip_isize_ios_and_exponent_8():
    data = text(70000, 9)
    for fmt, exponent in ((ds.GZIP, 15), (ds.IOS, 8), (ds.ZLIB, 8)):
        got, _ = stream(data, fmt, 7, exponent, [5000, 0, 1])
        z = b"".join(c for push in got for c in push)
        assert z == oracle.deflate(data, 7, fmt, exponent)
        if fmt == ds.GZIP:
            assert int.from_bytes(z[-4:], "little") == len(data)


def test_push_after_last_is_refused():
    d = ds.StreamingDeflator(ds.ZLIB, 4, 15, ds.CHUNK)
    d.push(b"abc", True)
    with pytest.raises(AssertionError):
        d.push(b"x")
