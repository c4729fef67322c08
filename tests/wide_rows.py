"""Rows long enough to wrap 32-bit arithmetic in the scanline kernels, with outputs known in closed form or cheap to get
from the oracle: test data only.

- Filter selection (filter_rows_kernel): a byte scores at most 128, so a row's score reaches 2^32 from pitch 2^25 on.
  The rows here are RGBA8, one row high, made of 0x80 bytes with a few edits that set the None score to exactly
  2^32 - 1, 2^32 or 2^32 + 1 (Up scores the same as None on a first row), while Sub keeps a score of a few hundred.
  The reference sums scores in 64 bits and picks Sub; a 32-bit sum sees None at 0, 1 or tied with Sub and picks None.
- Adam7 unfiltering (unfilter_generic_kernel): pass 7 has the full image width, so the pitch sw * volume / 8 passes 2^32
  bits-wise at width 2^26 for RGBA16 and 2^27 for RGBA8.
- Wavefront unfiltering (unfilter_wave_kernel): one-row RGBA16 images with pitches around 2^31.
"""
from __future__ import annotations

import numpy as np

BPP = 4                      # filter rows: RGBA8
FILTER_PITCHES = (2 ** 25 - 16, 2 ** 25, 2 ** 25 + 16)
ADAM7 = ((0, 0, 3, 3), (4, 0, 3, 3), (0, 4, 2, 3), (2, 0, 2, 2), (0, 2, 1, 2), (1, 0, 1, 1), (0, 1, 0, 1))
WAVE_PITCHES = (2 ** 31 - 16, 2 ** 31, 2 ** 31 + 16)


def scores(cur: np.ndarray, prev: np.ndarray, bpp: int) -> list[int]:
    """the five sum|int8| scores of PNG.Encoder.score (None, Sub, Up, Average, Paeth) as Python integers: numpy's
    version of the per-byte loop in test_emu_filter.scores"""
    x = cur.astype(np.int16)
    b = prev.astype(np.int16)
    a = np.zeros_like(x)
    c = np.zeros_like(x)
    a[bpp:], c[bpp:] = x[:-bpp], b[:-bpp]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    out = []
    for pred in (0, a, b, (a + b) >> 1, paeth):
        v = ((x - pred) & 0xFF).astype(np.uint8).view(np.int8)
        out.append(int(np.abs(v.astype(np.int16)).sum(dtype=np.int64)))
    return out


def pick(s: list[int], bits: int | None = None) -> int:
    """the first minimum (strict <, None..Paeth); with `bits`, of the scores reduced modulo 2^bits"""
    if bits is not None:
        s = [v & ((1 << bits) - 1) for v in s]
    return s.index(min(s))


def filter_row(pitch: int, dips: int = 0, tail: bytes = b"") -> np.ndarray:
    """0x80 bytes; `dips` of them lowered to 0x7f 8 bytes apart from byte 64 (each takes 1 from the None score and adds
    2 to Sub's), then the last bytes replaced by `tail`"""
    row = np.full(pitch, 0x80, np.uint8)
    row[64:64 + 8 * dips:8] = 0x7F
    if tail:
        row[pitch - len(tail):] = np.frombuffer(tail, np.uint8)
    return row


def filter_cases():
    """[(name, row, None score)]: single-row RGBA8 images (width = pitch / 4) whose None score sits at the 2^32 edge"""
    p0, p1, p2 = FILTER_PITCHES
    return [
        ("none-2^32-2048", filter_row(p0), 2 ** 32 - 2048),
        ("none-2^32-1", filter_row(p1, dips=1), 2 ** 32 - 1),
        ("none-up-tie-2^32", filter_row(p1), 2 ** 32),
        ("none-2^32+1", filter_row(p2, tail=b"\x01" + bytes(15)), 2 ** 32 + 1),
        ("wrapped-none-ties-sub", filter_row(p2, dips=512), 2 ** 32 + 1536),
    ]


def adam7_passes(w: int, h: int, volume: int):
    """[(pass, sub-image width, rows, pitch)] of the non-empty passes"""
    out = []
    for z, (bx, by, ex, ey) in enumerate(ADAM7):
        sw = (w + (1 << ex) - bx - 1) >> ex
        sh = (h + (1 << ey) - by - 1) >> ey
        if sw and sh:
            out.append((z, sw, sh, (sw * volume + 7) >> 3))
    return out


def row_passes(w: int, h: int, volume: int) -> list[int]:
    """the Adam7 pass (0..6) of every scanline, in stream order"""
    return [z for z, _, sh, _ in adam7_passes(w, h, volume) for _ in range(sh)]


def filtered_stream(w: int, h: int, volume: int, interlaced: bool, types, seed: int) -> bytearray:
    """seeded random scanlines behind filter-type bytes taken from `types` in turn (values above 4 are invalid filter
    bytes, which leave the row as it is)"""
    passes = adam7_passes(w, h, volume) if interlaced else [(0, w, h, (w * volume + 7) >> 3)]
    total = sum(sh * (pitch + 1) for _, _, sh, pitch in passes)
    data = np.random.default_rng(seed).integers(0, 256, total, dtype=np.uint8)
    at, k = 0, 0
    for _, _, sh, pitch in passes:
        for _ in range(sh):
            data[at] = types[k % len(types)]
            at += pitch + 1
            k += 1
    return bytearray(data.data)


def filtered_size(w: int, h: int, volume: int, interlaced: bool) -> int:
    if not interlaced:
        return h * (((w * volume + 7) >> 3) + 1)
    return sum(sh * (pitch + 1) for _, _, sh, pitch in adam7_passes(w, h, volume))
