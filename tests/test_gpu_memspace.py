"""Every batch entry point with host buffers (PNGB200_MEM_HOST: the library stages them through its own device
arenas) against the same batch with device buffers (PNGB200_MEM_DEVICE: torch tensors, used in place).  Both must
report the same statuses, error payloads, byte counts and checksums and write the same bytes.  Also: trimming a
context gives its big arenas back without changing what the next batch computes."""
from __future__ import annotations

import ctypes as C
import gzip
import zlib

import numpy as np
import pytest

import corpus
import pngio

pytestmark = pytest.mark.gpu


class Out:
    """an output buffer of n bytes (filled with 0xA5 before the call)"""

    def __init__(self, n: int):
        self.n = n


def scalars(s):
    """the descriptor's fields that are not pointers (nested structures and arrays included)"""
    out = {}
    for name, typ in s._fields_:
        if typ is C.c_void_p:
            continue
        v = getattr(s, name)
        out[name] = scalars(v) if isinstance(v, C.Structure) else list(v) if isinstance(v, C.Array) else v
    return out


def call(pngb200, ctx, fn, Desc, rows, memspace, *args, host=()):
    """ctx's `fn` over descriptors built from `rows`: per item a dict of field values, where bytes is an input buffer,
    Out(n) an output buffer and a callable fills the descriptor itself.  Buffers live in `memspace`, except the fields
    named in `host`, which the library always reads or writes on the host.  Returns per item (scalar fields, bytes of
    each output buffer)."""
    import torch
    descs = (Desc * len(rows))()
    keep, reads = [], []
    for i, row in enumerate(rows):
        mine = {}
        for name, v in row.items():
            if callable(v):
                v(descs[i], keep)
            elif isinstance(v, (bytes, Out)):
                data = v if isinstance(v, bytes) else b"\xa5" * v.n
                if memspace == pngb200.MEM_DEVICE and name not in host:
                    buf = torch.frombuffer(bytearray(data or b"\0"), dtype=torch.uint8).cuda()
                    addr = buf.data_ptr()
                    read = lambda buf=buf, n=len(data): buf[:n].cpu().numpy().tobytes()
                else:
                    buf = C.create_string_buffer(data, max(len(data), 1))
                    addr = C.addressof(buf)
                    read = lambda buf=buf, n=len(data): buf.raw[:n]
                keep.append(buf)
                setattr(descs[i], name, addr)
                if isinstance(v, Out):
                    mine[name] = read
            else:
                setattr(descs[i], name, v)
        reads.append(mine)
    torch.cuda.synchronize()
    ctx.check(getattr(ctx._lib, fn)(ctx.handle, descs, len(rows), *args, memspace))
    torch.cuda.synchronize()
    return [(scalars(descs[i]), {k: r() for k, r in reads[i].items()}) for i in range(len(rows))]


def same_both_ways(pngb200, ctx, fn, Desc, rows, *args, host=(), upto=None):
    """runs `rows` with host and with device buffers and asserts identical results.  Output bytes are compared in
    full for items that succeeded, or up to upto(fields) bytes when that is given (also for failed items)."""
    got = call(pngb200, ctx, fn, Desc, rows, pngb200.MEM_HOST, *args, host=host)
    dev = call(pngb200, ctx, fn, Desc, rows, pngb200.MEM_DEVICE, *args, host=host)
    for i, ((fh, oh), (fd, od)) in enumerate(zip(got, dev)):
        assert fh == fd, (fn, i)
        for name in oh:
            n = upto(fh) if upto else None
            if n is not None:
                assert oh[name][:n] == od[name][:n], (fn, i, name)
            elif fh["status"] == pngb200.OK:
                assert oh[name] == od[name], (fn, i, name)
    return got


def photos(specs):
    """[(image array, filtered, zlib stream)] for (w, h, seed, sixteen) specs"""
    out = []
    for w, h, seed, sixteen in specs:
        img = corpus.make("photo", w, h, seed, sixteen)
        filtered, z = corpus.zlib_png_stream(img, 8 if sixteen else 4, 6)
        out.append((img, filtered, z))
    return out


def spoiled(z: bytes) -> bytes:
    bad = bytearray(z)
    bad[-2] ^= 0x40   # the Adler-32 trailer
    return bytes(bad)


def test_inflate_batch(pngb200, ctx):
    rng = np.random.default_rng(11)
    (_, big, zbig), (_, small, zsmall) = photos([(300, 200, 1, False), (40, 20, 2, False)])
    text = bytes(rng.integers(97, 103, 5000, dtype=np.uint8))
    raw = zlib.compressobj(6, zlib.DEFLATED, -15)
    raw = raw.compress(big) + raw.flush()
    streams = [
        (zbig, big, pngb200.FORMAT_ZLIB), (zsmall, small, pngb200.FORMAT_ZLIB), (gzip.compress(big), big, pngb200.FORMAT_GZIP),
        (gzip.compress(text), text, pngb200.FORMAT_GZIP), (raw, big, pngb200.FORMAT_IOS), (zlib.compress(text, 9), text, pngb200.FORMAT_ZLIB),
        (zbig[: len(zbig) // 2], big, pngb200.FORMAT_ZLIB), (spoiled(zbig), big, pngb200.FORMAT_ZLIB), (spoiled(zsmall), small, pngb200.FORMAT_ZLIB),
    ]
    rows = [dict(src=s, src_len=len(s), dst=Out(len(plain) + 1024), dst_cap=len(plain) + 1024, format=f) for s, plain, f in streams]
    got = same_both_ways(pngb200, ctx, "pngb200_inflate_batch", pngb200.StreamDesc, rows, upto=lambda f: f["produced"])
    assert [f["status"] for f, _ in got[:6]] == [pngb200.OK] * 6
    assert got[0][1]["dst"][: len(big)] == big and got[3][1]["dst"][: len(text)] == text
    assert got[6][0]["status"] != pngb200.OK and got[7][0]["status"] == got[8][0]["status"] == pngb200.ERR_STREAM_CHECKSUM


def decode_rows(pngb200):
    rng = np.random.default_rng(12)
    rows = []
    for img, _, z in photos([(320, 240, 3, False), (64, 48, 4, True), (257, 33, 5, False)]):
        vol = 64 if img.shape[2] == 8 else 32
        rows.append(dict(idat=z, width=img.shape[1], height=img.shape[0], volume=vol, depth=vol // 4))
    # interlaced and sub-byte images go through the generic unfilter kernel
    for w, h, vol, depth, il in ((37, 29, 32, 8, 1), (61, 17, 2, 2, 0), (23, 40, 4, 4, 1)):
        filtered = bytearray(rng.integers(0, 256, pngb200.filtered_size(w, h, vol, bool(il)), dtype=np.uint8).tobytes())
        rows.append(dict(idat=zlib.compress(bytes(filtered)), width=w, height=h, volume=vol, depth=depth, interlaced=il))
    rows.append(dict(rows[0], idat=rows[0]["idat"][:-500]))     # truncated
    rows.append(dict(rows[2], idat=spoiled(rows[2]["idat"])))    # wrong checksum
    for r in rows:
        r["pixels"] = Out(pngb200.storage_size(r["width"], r["height"], r["volume"]))
        r["pixels_cap"] = r["pixels"].n
        r["idat_len"] = len(r["idat"])
    return rows


def test_decode_batch(pngb200, ctx):
    rows = decode_rows(pngb200)
    got = same_both_ways(pngb200, ctx, "pngb200_decode_batch", pngb200.ImageDesc, rows)
    assert [f["status"] for f, _ in got[:6]] == [pngb200.OK] * 6
    assert got[-2][0]["status"] != pngb200.OK and got[-1][0]["status"] == pngb200.ERR_STREAM_CHECKSUM
    assert got[0][1]["pixels"] == corpus.make("photo", 320, 240, 3).tobytes()


def test_unfilter_batch_wavefront_and_generic(pngb200, ctx):
    rows = []
    for r in decode_rows(pngb200)[:6]:
        r = dict(r, idat=zlib.decompress(r["idat"]))
        r["idat_len"] = len(r["idat"])
        rows.append(r)
    rows.append(dict(rows[0], idat=rows[0]["idat"] + b"\0\0\0", idat_len=rows[0]["idat_len"] + 3))   # extraneous data
    got = same_both_ways(pngb200, ctx, "pngb200_unfilter_batch", pngb200.ImageDesc, rows)
    assert [f["status"] for f, _ in got] == [pngb200.OK] * 6 + [pngb200.ERR_PNG_EXTRANEOUS_IMAGE_DATA]
    assert got[0][1]["pixels"] == corpus.make("photo", 320, 240, 3).tobytes()


def storages(pngb200):
    rows = []
    for w, h, vol, depth, il, seed in ((200, 120, 32, 8, 0, 1), (77, 31, 64, 16, 1, 2), (53, 9, 1, 1, 0, 3), (30, 30, 24, 8, 1, 4)):
        st = np.random.default_rng(seed).integers(0, 256, pngb200.storage_size(w, h, vol), dtype=np.uint8).tobytes()
        rows.append(dict(st=st, width=w, height=h, volume=vol, depth=depth, interlaced=il))
    return rows


def test_filter_batch(pngb200, ctx):
    rows = []
    for s in storages(pngb200):
        n = pngb200.filtered_size(s["width"], s["height"], s["volume"], bool(s["interlaced"]))
        rows.append(dict(pixels=s["st"], pixels_len=len(s["st"]), filtered=Out(n), filtered_cap=n, width=s["width"],
                         height=s["height"], volume=s["volume"], depth=s["depth"], interlaced=s["interlaced"]))
    got = same_both_ways(pngb200, ctx, "pngb200_filter_batch", pngb200.FilterDesc, rows)
    assert all(f["status"] == pngb200.OK and f["produced"] == r["filtered_cap"] for (f, _), r in zip(got, rows))


def test_deflate_batch(pngb200, ctx):
    rng = np.random.default_rng(13)
    data = [photos([(120, 80, 6, False)])[0][1], bytes(rng.integers(97, 100, 20000, dtype=np.uint8)), b"", bytes(rng.integers(0, 256, 3000, dtype=np.uint8))]
    rows = []
    for k, (d, level, fmt) in enumerate(zip(data, (9, 4, 6, 1), (pngb200.FORMAT_ZLIB, pngb200.FORMAT_GZIP, pngb200.FORMAT_IOS, pngb200.FORMAT_ZLIB))):
        cap = pngb200.lib().pngb200_deflate_bound(len(d))
        rows.append(dict(src=d, src_len=len(d), dst=Out(cap), dst_cap=cap, format=fmt, level=level, exponent=15 - k))
    got = same_both_ways(pngb200, ctx, "pngb200_deflate_batch", pngb200.DeflateDesc, rows, upto=lambda f: f["produced"])
    assert all(f["status"] == pngb200.OK for f, _ in got)
    assert zlib.decompress(got[0][1]["dst"][: got[0][0]["produced"]]) == data[0]


def test_encode_batch(pngb200, ctx):
    rows = []
    for s, level in zip(storages(pngb200), (9, 6, 3, 1)):
        cap = pngb200.lib().pngb200_deflate_bound(pngb200.filtered_size(s["width"], s["height"], s["volume"], bool(s["interlaced"])))
        rows.append(dict(pixels=s["st"], pixels_len=len(s["st"]), idat=Out(cap), idat_cap=cap, width=s["width"], height=s["height"],
                         volume=s["volume"], depth=s["depth"], interlaced=s["interlaced"], format=pngb200.FORMAT_ZLIB, level=level))
    got = same_both_ways(pngb200, ctx, "pngb200_encode_batch", pngb200.EncodeDesc, rows, upto=lambda f: f["produced"])
    assert all(f["status"] == pngb200.OK for f, _ in got)


def colour_formats():
    """(color, depth, bgr, key, palette) covering every colour type, a key, bgr and a palette"""
    pal = bytes(np.random.default_rng(14).integers(0, 256, 4 * 16, dtype=np.uint8))
    return [(6, 8, False, None, None), (2, 16, False, (3, 4, 5), None), (0, 4, False, (2,), None), (4, 16, False, None, None),
            (3, 4, False, None, pal), (6, 8, True, None, None), (0, 16, False, None, None)]


def sample_top(color, depth):
    """one more than the largest storage byte of a valid image: palette indices stay inside the 16-entry palette"""
    return 16 if color == 3 else 1 << depth if depth < 8 else 256


def fill_format(pngb200, color, depth, bgr, key, palette):
    return lambda d, keep: pngb200._fill_format(d.format, keep, color, depth, bgr, key, palette)


@pytest.mark.parametrize("target", [0, 1, 3, 4, 7, 8, 11])
def test_unpack_and_pack_batch(pngb200, ctx, target):
    rng = np.random.default_rng(15 + target)
    tb = pngb200._TARGET_BYTES[target]
    unpack, pack = [], []
    for k, (color, depth, bgr, key, pal) in enumerate(colour_formats()):
        count = 97 + 61 * k
        n = count * pngb200._CHANNELS[color] * (2 if depth == 16 else 1)
        st = rng.integers(0, sample_top(color, depth), n, dtype=np.uint8).tobytes()
        fmt = fill_format(pngb200, color, depth, bgr, key, pal)
        unpack.append(dict(storage=st, storage_len=n, pixels=Out(count * tb), pixels_len=count * tb, count=count, format=fmt))
        px = rng.integers(0, 256, count * tb, dtype=np.uint8).tobytes()
        pack.append(dict(pixels=px, pixels_len=len(px), storage=Out(n), storage_len=n, count=count, format=fmt))
    alpha = pngb200.ALPHA_PREMULTIPLIED if target < pngb200.TARGET_V8 else pngb200.ALPHA_ASIS
    got = same_both_ways(pngb200, ctx, "pngb200_unpack_batch", pngb200.ColorDesc, unpack, target, alpha)
    assert all(f["status"] == pngb200.OK for f, _ in got)
    same_both_ways(pngb200, ctx, "pngb200_pack_batch", pngb200.ColorDesc, pack, target)


def png_files():
    rng = np.random.default_rng(16)
    files = []
    for img, _, z in photos([(300, 200, 7, False), (45, 38, 8, True)]):
        files.append(pngio.write(img.shape[1], img.shape[0], 8 if img.shape[2] == 4 else 16, 6, z, idat_chunk=4096))
    filtered = rng.integers(0, 256, (16 * 4 // 8 + 1) * 16, dtype=np.uint8)
    filtered[:: 16 * 4 // 8 + 1] %= 5
    pal = bytes(rng.integers(0, 256, 3 * 16, dtype=np.uint8))
    files.append(pngio.write(16, 16, 4, 3, zlib.compress(filtered.tobytes()), palette=pal, trns=b"\x10\x80"))
    hurt = bytearray(files[0])
    hurt[len(hurt) // 2] ^= 0x10                                   # a bad CRC inside the IDAT run
    files.append(bytes(hurt))
    files.append(files[1][: len(files[1]) - 30])                  # truncated before IEND
    files.append(files[0][:33] + pngio.chunk(b"IEND", b""))        # no IDAT
    return files


def test_png_decode_batch(pngb200, ctx):
    files = png_files()
    probe = pngb200.png_inspect(files)
    rows = [dict(file=f, file_len=len(f), pixels=Out(max(p.width * p.height * 8, 1)), pixels_cap=max(p.width * p.height * 8, 1))
            for f, p in zip(files, probe)]
    got = same_both_ways(pngb200, ctx, "pngb200_png_decode_batch", pngb200.PngDesc, rows, host=("file",))
    assert [f["status"] == pngb200.OK for f, _ in got] == [True, True, True, False, False, False]
    assert got[3][0]["status"] == pngb200.ERR_LEX_INVALID_CHUNK_CHECKSUM


def test_png_encode_batch(pngb200, ctx):
    rows = []
    rng = np.random.default_rng(17)
    for k, (color, depth, bgr, key, pal) in enumerate(colour_formats()):
        w, h, il = 31 + 20 * k, 17 + 3 * k, k % 2
        n = pngb200.storage_size(w, h, depth * pngb200._CHANNELS[color])
        st = rng.integers(0, sample_top(color, depth), n, dtype=np.uint8).tobytes()
        f = pngb200.PixelFormat()
        pngb200._fill_format(f, [], color, depth, bgr, key, pal)
        cap = pngb200.lib().pngb200_png_encode_bound(w, h, C.byref(f), il, 1000)
        rows.append(dict(pixels=st, pixels_len=n, width=w, height=h, format=fill_format(pngb200, color, depth, bgr, key, pal),
                         interlaced=il, level=(9, 6, 1)[k % 3], idat_chunk=1000, file=Out(cap), file_cap=cap))
    got = same_both_ways(pngb200, ctx, "pngb200_png_encode_batch", pngb200.PngEncodeDesc, rows, host=("file",),
                         upto=lambda f: f["produced"])
    assert all(f["status"] == pngb200.OK for f, _ in got)
    back = pngb200.png_decode_batch(ctx, [o["file"][: f["produced"]] for f, o in got])
    assert all(b.status == pngb200.OK for b in back)
    assert back[0].storage == rows[0]["pixels"] and back[1].storage == rows[1]["pixels"]


def run_everything(pngb200, ctx):
    """one batch through each family of arenas the trim releases; returns everything it computed"""
    rows = decode_rows(pngb200)
    out = [call(pngb200, ctx, "pngb200_decode_batch", pngb200.ImageDesc, rows, pngb200.MEM_HOST)]
    big = photos([(300, 200, 1, False)])[0][1]
    streams = pngb200.inflate_batch(ctx, [zlib.compress(big), gzip.compress(big)], [pngb200.FORMAT_ZLIB, pngb200.FORMAT_GZIP])
    out.append([(st, data, d.checksum, d.produced) for st, data, d in streams])
    out.append(pngb200.deflate_batch(ctx, [big[:50000]], level=9))
    out.append([(im.status, im.err_a, im.err_b, im.storage) for im in pngb200.png_decode_batch(ctx, png_files())])
    img = corpus.make("photo", 90, 60, 9)
    out.append(pngb200.png_encode_batch(ctx, [dict(storage=img.tobytes(), width=90, height=60, color=6, depth=8)], level=6))
    return out


def test_trim_then_same_batch_again(pngb200):
    ctx = pngb200.Context(0)
    try:
        first = run_everything(pngb200, ctx)
        hist = ctx.filter_histogram()
        ctx.trim()
        assert ctx.filter_histogram() == hist   # the histogram lives in an arena the trim keeps
        assert run_everything(pngb200, ctx) == first
        ctx.trim()
        ctx.trim()
        assert run_everything(pngb200, ctx) == first
    finally:
        ctx.close()


def test_trim_while_a_decode_batch_is_pending(pngb200):
    ctx = pngb200.Context(0)
    try:
        rows = decode_rows(pngb200)[:3]
        descs = (pngb200.ImageDesc * len(rows))()
        keep = []
        for i, r in enumerate(rows):
            src = C.create_string_buffer(r["idat"], len(r["idat"]))
            dst = C.create_string_buffer(r["pixels_cap"])
            keep.append((src, dst))
            descs[i].idat, descs[i].idat_len = C.addressof(src), len(r["idat"])
            descs[i].pixels, descs[i].pixels_cap = C.addressof(dst), r["pixels_cap"]
            descs[i].width, descs[i].height, descs[i].volume, descs[i].depth = r["width"], r["height"], r["volume"], r["depth"]
        ctx.check(ctx._lib.pngb200_decode_batch_enqueue(ctx.handle, descs, len(rows), pngb200.MEM_HOST))
        assert ctx._lib.pngb200_ctx_trim(ctx.handle) == pngb200.ERR_BAD_ARGUMENT
        assert b"pending" in ctx._lib.pngb200_last_error(ctx.handle)
        ctx.check(ctx._lib.pngb200_decode_batch_finish(ctx.handle, descs, len(rows)))
        assert [descs[i].status for i in range(len(rows))] == [pngb200.OK] * 3
        assert keep[0][1].raw[: rows[0]["pixels_cap"]] == corpus.make("photo", 320, 240, 3).tobytes()
        ctx.trim()
    finally:
        ctx.close()
