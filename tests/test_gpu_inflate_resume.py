"""The streaming inflator on the H100 resumes inside a DEFLATE block: pushes of any size decode each input bit about once.
Long single-block streams (fixed and dynamic Huffman, at least 16 MiB of output) are pushed in 65 544-byte, 8 KiB,
7-byte and uneven pieces in the zlib, gzip and raw formats.  After every push the bytes pulled are the stream's complete
symbols so far (zlib's incremental inflate releases exactly those; the oracle's one-shot inflate of a few prefixes
confirms it), and the handle's work counters (Inflator.stats) stay linear in the stream's length: the parent commit
decoded the block in flight again from its header on every push.  An 8K level-9 PNG file pushed chunk by chunk through
PngContext decodes to png_decode_batch's storage, and its twin inflator's work is linear too.

Each test states its peak device memory and skips, naming the number, when that much is not free (the GPU is shared)."""
from __future__ import annotations

import zlib

import numpy as np
import pytest

import corpus
import deflate_craft as dc
import pngio
from oracle import oracle

pytestmark = pytest.mark.gpu
GiB = 1 << 30
WV_BITS = 65536          # input bits of one wave of the ring kernel (csrc/inflate_stream.cuh)
HEADER_BITS = 4600       # more than the longest dynamic block header (3 + 14 + 19 * 3 + 316 * 14 bits)
FORMATS = {"zlib": (0, 15), "ios": (1, -15), "gzip": (2, 31)}   # pngb200 format, zlib wbits


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


_STREAMS = {}


def long_block(kind: str):
    """(writer, plain): ONE fixed or dynamic block of more than 16 MiB of output: literal runs and copies of every
    length at distances up to 32 768"""
    if kind not in _STREAMS:
        rng = np.random.default_rng(16 + (kind == "dynamic"))
        w = dc.Writer()
        tokens, n = [rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes()], 40_000
        while n < (16 << 20) + 65536:
            run = rng.integers(0, 256, int(rng.integers(10, 90)), dtype=np.uint8).tobytes()
            length = int(rng.integers(3, 259))
            tokens += [run, (length, int(rng.integers(1, 32769)), length == 258 and n % 2 == 1)]
            n += len(run) + length
        if kind == "fixed":
            w.fixed(tokens, final=True)
        else:
            w.dynamic(tokens, *dc._freq_lengths(tokens), final=True)
        assert len(w.blocks) == 1
        _STREAMS[kind] = w
    return _STREAMS[kind]


def pieces(stream: bytes, how: str):
    if how == "65544":
        return [stream[i:i + 65544] for i in range(0, len(stream), 65544)]
    if how == "8k":
        return [stream[i:i + 8192] for i in range(0, len(stream), 8192)]
    if how == "7":   # a prefix in 7-byte pieces, then the rest at once
        head = 7 * 28_572
        return [stream[i:i + 7] for i in range(0, head, 7)] + [stream[head:]]
    rng = np.random.default_rng(len(stream))
    out, at = [], 0
    while at < len(stream):
        n = int(rng.choice([1, 13, 4096, 60_000, 70_000, 300_000, 1_500_000]))
        out.append(stream[at:at + n])
        at += n
    return out


def wave_output_bound(stream: bytes, plain: bytes) -> int:
    """bytes one wave's input decodes to: twice the stream's mean, for these streams whose tokens are drawn uniformly"""
    return 2 * len(plain) * WV_BITS // (8 * len(stream)) + 258


def check_linear(stats: dict, stream: bytes, plain: bytes, pushes: int, stored: int = 0):
    wave_out = wave_output_bound(stream, plain)
    assert stats["bits"] <= 8 * len(stream) + pushes * (HEADER_BITS + WV_BITS), (stats, pushes)
    assert stats["serial_bytes"] <= pushes * wave_out + stored, (stats, pushes, wave_out)
    assert stats["bytes"] <= len(plain) + pushes * wave_out, (stats, pushes)


@pytest.mark.parametrize("how", ["65544", "8k", "7", "uneven"])
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("kind", ["fixed", "dynamic"])
def test_long_block(pngb200, budget, kind, fmt, how):
    """peak 0.2 GiB: the input, a doubling output buffer of the handle and the checksum pass's partial sums"""
    ctx = budget(0.2)
    w = long_block(kind)
    stream, plain, _ = w.finish({"zlib": "zlib", "ios": "raw", "gzip": "gzip"}[fmt])
    fcode, wbits = FORMATS[fmt]
    assert len(plain) >= 16 << 20
    ps = pieces(stream, how)
    z = pngb200.Inflator(ctx, fcode)
    ref = zlib.decompressobj(wbits)
    got, want = 0, 0
    probes = {len(ps) // 3, len(ps) // 2}
    at = 0
    try:
        for i, p in enumerate(ps):
            st = z.push(p)
            at += len(p)
            want += len(ref.decompress(p))
            out = z.pull_all()
            assert plain[got:got + len(out)] == out, i
            got += len(out)
            assert got == want, (i, got, want)
            assert st == (0 if i == len(ps) - 1 else 1), (i, st)
            if i in probes:   # the reference's own prefix semantics
                ost, obytes, _ = oracle.inflate(stream[:at], fcode, len(plain))
                assert (ost, len(obytes)) == (1, got)
        assert got == len(plain)
        check_linear(z.stats(), stream, plain, len(ps))
    finally:
        z.close()


def test_errors_after_a_resume_point(pngb200, budget):
    """peak 0.1 GiB: a defect several pushes into a stream (invalid distance and literal/length codes) gives
    the oracle's status and payload, from the ring kernel and from the serial decoder"""
    ctx = budget(0.1)
    for name in ("bad_hdist31_used", "bad_one_code_unassigned", "bad_fixed_lit286"):
        case = dc.build(name, 600_000, seed=5)
        stream, _, _ = case.stream("zlib")
        for step in (70_001, 5_003):
            z = pngb200.Inflator(ctx, 0)
            st, payload, n = 1, None, 0
            for at in range(0, len(stream), step):
                try:
                    st = z.push(stream[at:at + step])
                except pngb200.PNGB200Error as e:
                    st, payload = e.status, e.payload
                    break
                n += 1
            assert n >= 2 and (st, payload) == (case.status, case.err), (name, step, n, st, payload)
            z.close()


def test_whole_8k_file(pngb200, budget):
    """peak 1.0 GiB: an 8K RGBA8 level-9 file pushed as its 65 544-byte IDAT chunks through a PngContext (host storage)
    and a twin Inflator: png_decode_batch's storage, and linear work"""
    ctx = budget(1.0)
    W, H = 7680, 4320
    img = corpus.make("photo", W, H, 11).tobytes()
    f = oracle.png_compress(img, W, H, oracle.make_format(6, 8), False, 9, 65544)
    chunks = pngio.idat_chunks(f)
    (dec,) = pngb200.png_decode_batch(ctx, [f])
    assert dec.status == 0 and dec.storage == img
    c = pngb200.PngContext(ctx, W, H, 32, 8, False)
    twin = pngb200.Inflator(ctx)
    try:
        for p in chunks:
            before = ctx.launches
            twin.push(p)
            assert ctx.launches - before <= 4
            c.push(p, False)
        c.end()
        assert c.storage() == dec.storage
        stream = b"".join(chunks)
        plain = twin.pull_all()
        assert len(plain) == oracle.filtered_size(W, H, 32)
        check_linear(twin.stats(), stream, plain, len(chunks))
    finally:
        c.close()
        twin.close()
