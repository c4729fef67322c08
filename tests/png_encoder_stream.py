"""The online encoder's restatement on the CPU (test infrastructure only): PNG.Image.compress(stream:level:hint:) as
PNG.Encoder.pull runs it when the storage rows arrive over time.  The filtered stream of oracle.png_filter is cut into
scanlines and pushed one scanline at a time into the streaming restatement of LZ77.Deflator (deflate_stream), with
pop() drained before each scanline is collected; pull() asks for the first scanline the rows so far do not complete,
so a push makes available exactly what the reference has written by then.  The push that brings the last row ends the
stream: push([], last: true), pull() until nil, IEND."""
from __future__ import annotations

import deflate_stream as ds
import pngio

# PNG.adam7: (base x, base y, exponent x, exponent y)
ADAM7 = ((0, 0, 3, 3), (4, 0, 3, 3), (0, 4, 2, 3), (2, 0, 2, 2), (0, 2, 1, 2), (1, 0, 1, 1), (0, 1, 0, 1))
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def volume(fields) -> int:
    return fields["depth"] * CHANNELS[fields["color"]]


def scanlines(w: int, h: int, vol: int, interlaced: bool) -> list:
    """[(storage row the scanline needs last, start, end)] in stream order"""
    out, at = [], 0
    for bx, by, ex, ey in (ADAM7 if interlaced else ((0, 0, 0, 0),)):
        sw, sh = (w + (1 << ex) - bx - 1) >> ex, (h + (1 << ey) - by - 1) >> ey
        if sw <= 0 or sh <= 0:
            continue
        pitch = (sw * vol + 7) >> 3
        for y in range(sh):
            out.append((by + (y << ey), at, at + pitch + 1))
            at += pitch + 1
    return out


def head(file: bytes) -> bytes:
    """the bytes in front of the first IDAT chunk"""
    return file[: file.index(b"IDAT") - 4]


def pieces(orc, storage: bytes, w: int, h: int, fields: dict, interlaced: bool, level: int, idat_chunk: int,
           schedule) -> list:
    """The pieces available after each push of `schedule` (storage rows per push, summing to h): the head with the
    first push, then framed IDAT chunks, then IEND with the push that brings the last row."""
    fmt = orc.make_format(**fields)
    vol = volume(fields)
    filtered = orc.png_filter(storage, w, h, vol, fields["depth"], interlaced)
    lines = scanlines(w, h, vol, interlaced)
    assert lines[-1][2] == len(filtered)
    d = ds.StreamingDeflator(ds.IOS if fields.get("bgr") else ds.ZLIB, level, 15, idat_chunk)
    top = head(orc.png_compress(storage, w, h, fmt, interlaced, level, idat_chunk=idat_chunk))
    out, k, rows = [], 0, 0
    for n in schedule:
        rows += n
        got = [top] if not out else []
        while True:
            got += [pngio.chunk(b"IDAT", c) for c in ds.drain(d)]   # pop() before each collect
            if k == len(lines) or lines[k][0] >= rows:
                break
            d.push(filtered[lines[k][1]: lines[k][2]])
            k += 1
        if rows == h:
            d.push(b"", True)
            got += [pngio.chunk(b"IDAT", c) for c in ds.drain(d, True)] + [pngio.chunk(b"IEND", b"")]
        out.append(got)
    assert rows == h
    d.close()
    return out


def schedule(h: int, kind) -> list:
    """rows per push: 'rows' one at a time, 'all' in one push, an int for bands of that many rows, or a list of band
    sizes cycled (zeros included) until the image is complete"""
    if kind == "rows":
        return [1] * h
    if kind == "all":
        return [h]
    sizes = [kind] if isinstance(kind, int) else list(kind)
    out, left, i = [], h, 0
    while left:
        n = min(left, sizes[i % len(sizes)])
        out.append(n)
        left -= n
        i += 1
    return out
