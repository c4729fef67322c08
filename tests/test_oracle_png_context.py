"""The oracle's restatement of online decoding (oracle/png_context.c: PNG.Context, PNG.Decoder.push, PNG.Image.overdraw)
against the oracle's one-shot decode, an independent Python model of overdraw, and hand-checked cases."""
from __future__ import annotations

import zlib

import pytest

import pngio
from oracle import oracle
from png_context_cases import (GOLDEN, OracleContext, OverdrawModel, geometry, goldens, none_stream, random_storage,
                               row_ends, stored_prefix, stored_zlib)

GOLDENS = goldens()


def run(png, pieces, overdraw=False):
    """push every piece, then end(); (first error or end()'s status, storage, statuses)"""
    c = OracleContext(**geometry(png))
    sts = [c.push(p, overdraw) for p in pieces]
    errs = [s for s in sts if s < 0]
    st = errs[0] if errs else c.end()
    return st, c.storage(), sts


@pytest.mark.parametrize("name,data", GOLDENS, ids=[n for n, _ in GOLDENS])
def test_goldens_end_in_the_one_shot_decode(name, data):
    """one push of the whole IDAT run, and the file's own IDAT chunks one by one, with and without overdraw, end in
    orc_png_decode's storage and status"""
    png = pngio.parse(data)
    st, storage, _ = oracle.png_decode(png.idat, png.width, png.height, png.volume, png.depth, png.interlaced, png.fmt)
    for pieces in ([png.idat], pngio.idat_chunks(data)):
        for overdraw in (False, True):
            got_st, got, sts = run(png, pieces, overdraw)
            assert (got_st, got) == (st, storage), (name, len(pieces), overdraw)
            assert all(s == 0 for s in sts)


@pytest.mark.parametrize("volume,depth", [(1, 1), (2, 2), (4, 4), (8, 8), (16, 16), (32, 8), (48, 16)])
def test_overdraw_matches_python_model_after_every_push(volume, depth):
    """Adam7 images 1x1 ... 17x17, pushed 7 bytes at a time: after every push the storage equals an independent model of
    assign + overdraw over the rows the one-shot inflate of the pushed prefix makes available"""
    sizes = [(w, h) for w in range(1, 18) for h in range(1, 18)]
    if volume > 16:
        sizes = sizes[::5]
    for w, h in sizes:
        final = random_storage(w, h, volume, depth, w * 100 + h)
        filtered = oracle.png_filter(final, w, h, volume, depth, True)
        idat = zlib.compress(filtered, 9) if (w + h) % 2 else stored_zlib(filtered, 37)
        c = OracleContext(w, h, volume, depth, True)
        model = OverdrawModel(w, h, volume, True, final)
        ends, done = row_ends(w, h, volume, True), 0
        for at in range(0, len(idat), 7):
            assert c.push(idat[at:at + 7], True) == 0
            avail = len(oracle.inflate(idat[:at + 7], oracle.ZLIB)[1])
            while done < len(ends) and ends[done][2] <= avail:
                model.row(ends[done][0], ends[done][1], True)
                done += 1
            assert c.storage() == model.storage(), (w, h, at)
        assert c.end() == 0 and c.storage() == final


def test_hand_checked_9x9():
    """9x9 Adam7 RGBA8: once pass 0's first row has arrived, the top-left 8x8 block is pixel (0, 0) and rows 0-7 of
    column 8 are pixel (8, 0); nothing else is written"""
    w = h = 9
    final = random_storage(w, h, 32, 8, 9)
    stream = none_stream(final, w, h, 32, 8, True)
    idat = stored_zlib(stream)
    c = OracleContext(w, h, 32, 8, True)
    assert c.push(idat[:stored_prefix(9)], True) == 0      # filter byte + 2 pixels
    assert c.progress()[:2] == (0, 1) and c.progress()[4:] == (0, 8)
    px = lambda b, x, y: b[4 * (y * w + x):4 * (y * w + x) + 4]  # noqa: E731
    got = c.storage()
    for y in range(9):
        for x in range(9):
            want = px(final, 0, 0) if x < 8 and y < 8 else px(final, 8, 0) if y < 8 else bytes(4)
            assert px(got, x, y) == want, (x, y)


def test_statuses():
    w, h = 20, 11
    final = random_storage(w, h, 24, 8, 3)
    filtered = oracle.png_filter(final, w, h, 24, 8, False)
    idat = zlib.compress(filtered, 6)
    # -49 after the trailer, even for an empty push; end() before (-50) and after (OK) the trailer
    c = OracleContext(w, h, 24, 8)
    assert c.push(idat[:-3]) == 0 and c.end() == oracle.ERR_PNG_INCOMPLETE_DATASTREAM
    assert c.progress()[0] == 7 and c.storage() == final
    assert c.push(idat[-3:]) == 0 and c.end() == 0 and c.progress()[3] == 1
    assert c.push(b"") == oracle.ERR_PNG_EXTRANEOUS_COMPRESSED_DATA
    # -48 in the completing push, and in a later one that brings more filtered bytes
    extra = stored_zlib(filtered + b"\x00" * 120, 50)
    c = OracleContext(w, h, 24, 8)
    cut = stored_prefix((len(filtered) + 50) // 50 * 50, 50)      # the next byte is a block header
    assert c.push(extra[:cut]) == oracle.ERR_PNG_EXTRANEOUS_IMAGE_DATA and c.storage() == final
    assert c.push(extra[cut:cut + 1]) == 0      # no filtered byte in it
    assert c.push(extra[cut + 1:cut + 10]) == oracle.ERR_PNG_EXTRANEOUS_IMAGE_DATA
    # a corrupted byte: the one-shot status, storage as the previous push left it, sticky
    bad = bytearray(idat)
    bad[len(bad) // 2] ^= 0x40
    c = OracleContext(w, h, 24, 8)
    st_ref = oracle.inflate(bytes(bad), oracle.ZLIB)[0]
    assert st_ref < 0
    st = 0
    for at in range(0, len(bad), 16):
        before = c.storage()
        st = c.push(bytes(bad[at:at + 16]))
        if st < 0:
            assert c.storage() == before
            break
    assert st == st_ref and c.push(b"x") == st and c.error()[0] == st


def test_stored_block_bytes_arrive_as_pushed():
    """z00n2c08 (level 0) pushed in small pieces: rows are assigned while their stored block is still arriving"""
    data = open(f"{GOLDEN}/pngsuite/z00n2c08.png", "rb").read()
    png = pngio.parse(data)
    c = OracleContext(png.width, png.height, png.volume, png.depth, png.interlaced)
    rows = []
    for at in range(0, len(png.idat), 100):
        assert c.push(png.idat[at:at + 100]) == 0
        rows.append(c.progress()[1] if c.progress()[0] == 0 else png.height)
    assert rows[1] > 0 and len(set(rows)) > len(rows) // 2, rows
