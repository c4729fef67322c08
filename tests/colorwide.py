"""Test infrastructure: a Python restatement of every colour target, T = UInt8 ... UInt64.

The C oracle (oracle/png_color.c) restates the 8- and 16-bit RGBA / VA targets.  This module restates
all twelve pngb200 targets with Python integers, so the 64-bit premultiply / straighten products are
exact: image.unpack(as: RGBA<T> / VA<T> / T) and PNG.Image(packing:) with the default deindexer /
indexer (Sources/PNG/PNG.Image.swift:681-833, 1126-1145, ColorTargets/PNG.RGBA.swift:115-206,
PNG.swift:54-117, 255-261, 494-523, 1063-1097).  tests/test_color_wide_ref.py pins it to the C oracle
on the four targets they share and to the reference's goldens on the rest.
"""
import numpy as np

ERR_PALETTE_INDEX = -51
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# target -> (component bits, shape)
TARGETS = {0: (8, "rgba"), 1: (16, "rgba"), 2: (8, "va"), 3: (16, "va"),
           4: (32, "rgba"), 5: (64, "rgba"), 6: (32, "va"), 7: (64, "va"),
           8: (8, "v"), 9: (16, "v"), 10: (32, "v"), 11: (64, "v")}
NEW_TARGETS = list(range(4, 12))
WIDTH = {"rgba": 4, "va": 2, "v": 1}
DTYPE = {8: np.dtype("u1"), 16: np.dtype("<u2"), 32: np.dtype("<u4"), 64: np.dtype("<u8")}
AS_BITS = {3: 8, 4: 8, 5: 16, 6: 16, 7: 32, 8: 32}  # alpha mode -> U of premultiplied(as: U)


def tmax(bits: int) -> int:
    return (1 << bits) - 1


def target_bytes(target: int) -> int:
    bits, shape = TARGETS[target]
    return bits // 8 * WIDTH[shape]


def valid(target: int, mode: int) -> bool:
    """the combinations pngb200_unpack_batch accepts"""
    if target not in TARGETS or not 0 <= mode <= 8:
        return False
    bits, shape = TARGETS[target]
    if shape == "v":
        return mode == 0
    return mode < 3 or bits > AS_BITS[mode]


def modes(target: int) -> list:
    return [m for m in range(9) if valid(target, m)]


def premultiply(c, a, bits: int):
    """PNG.premultiply (PNG.swift:54-66): (c * a + T.max >> 1) / T.max; ints or object arrays"""
    m = tmax(bits)
    return (c * a + (m >> 1)) // m


def straighten(p, a, bits: int):
    """PNG.straighten (PNG.swift:100-120), saturating at T.max where the reference traps"""
    m = tmax(bits)
    if isinstance(a, np.ndarray):
        q = (m * p + (a >> 1)) // np.where(a == 0, 1, a)
        return np.where(a == 0, p, np.minimum(q, m))
    return p if a == 0 else min((m * p + (a >> 1)) // a, m)


def _widen(v: np.ndarray, depth: int, bits: int) -> np.ndarray:
    if bits >= depth:
        return v * np.uint64(tmax(bits) // tmax(depth))
    return v >> np.uint64(depth - bits)


def _narrow(v: np.ndarray, bits: int, depth: int) -> np.ndarray:
    if bits >= depth:
        return v >> np.uint64(bits - depth)
    return v * np.uint64(tmax(depth) // tmax(bits))


def _samples(storage: bytes, color: int, depth: int) -> np.ndarray:
    b = np.frombuffer(storage, np.uint8)
    if depth == 16:
        b = b.reshape(-1, 2).astype(np.uint64)
        raw = b[:, 0] << np.uint64(8) | b[:, 1]
    else:
        raw = b.astype(np.uint64)
    return raw.reshape(-1, CHANNELS[color])


def rgba(storage: bytes, bits: int, color: int, depth: int, bgr=False, key=None, palette=None):
    """(status, r, g, b, a) of every pixel in T's range, before any alpha mode"""
    raw = _samples(storage, color, depth)
    full = np.full(len(raw), tmax(bits), np.uint64)
    if color == 3:
        pal = np.frombuffer(bytes(palette), np.uint8).reshape(-1, 4).astype(np.uint64)
        idx = raw[:, 0].astype(np.int64)
        if len(idx) and idx.max() >= len(pal):
            return ERR_PALETTE_INDEX, None
        e = _widen(pal[idx], 8, bits)
        return 0, (e[:, 0], e[:, 1], e[:, 2], e[:, 3])
    if color in (0, 4):
        v = _widen(raw[:, 0], depth, bits)
        if color == 4:
            a = _widen(raw[:, 1], depth, bits)
        else:
            a = np.where(raw[:, 0] == key[0], np.uint64(0), full) if key is not None else full
        return 0, (v, v, v, a)
    c = [_widen(raw[:, k], depth, bits) for k in range(3)]
    r, g, b = (c[2], c[1], c[0]) if bgr else (c[0], c[1], c[2])
    if color == 6:
        a = _widen(raw[:, 3], depth, bits)
    elif key is not None:
        hit = (raw[:, 0] == key[0]) & (raw[:, 1] == key[1]) & (raw[:, 2] == key[2])
        a = np.where(hit, np.uint64(0), full)
    else:
        a = full
    return 0, (r, g, b, a)


def alpha(r, g, b, a, bits: int, mode: int):
    """the alpha modes on object arrays (Python integers, so 128-bit products are exact)"""
    if mode == 0:
        return r, g, b, a
    r, g, b, a = (x.astype(object) for x in (r, g, b, a))
    if mode in (1, 2):
        op = premultiply if mode == 1 else straighten
        return op(r, a, bits), op(g, a, bits), op(b, a, bits), a
    u = AS_BITS[mode]
    shift = bits - u
    q = tmax(bits) // (tmax(bits) >> shift)
    au = a >> shift
    op = premultiply if mode % 2 == 1 else straighten
    return op(r >> shift, au, u) * q, op(g >> shift, au, u) * q, op(b >> shift, au, u) * q, au * q


def unpack(storage: bytes, target: int, mode: int = 0, *, color, depth, bgr=False, key=None, palette=None):
    """(status, bytes of native little-endian T components); bytes is None on a palette error"""
    assert valid(target, mode), (target, mode)
    bits, shape = TARGETS[target]
    st, px = rgba(storage, bits, color, depth, bgr, key, palette)
    if st:
        return st, None
    r, g, b, a = alpha(*px, bits, mode)
    cols = {"rgba": (r, g, b, a), "va": (r, a), "v": (r,)}[shape]
    return 0, np.stack([np.asarray(c).astype(np.uint64) for c in cols], axis=1).astype(DTYPE[bits]).tobytes()


def pack(pixels: bytes, target: int, *, color, depth, bgr=False, key=None, palette=None) -> bytes:
    """PNG.Image(packing:) storage of a [RGBA<T>] / [VA<T>] / [T] array"""
    bits, shape = TARGETS[target]
    arr = np.frombuffer(pixels, DTYPE[bits]).astype(np.uint64).reshape(-1, WIDTH[shape])
    full = np.full(len(arr), tmax(bits), np.uint64)
    if shape == "rgba":
        r, g, b, a = arr[:, 0], arr[:, 1], arr[:, 2], arr[:, 3]
    else:  # VA: (v, a); scalar: (v, T.max)
        r = g = b = arr[:, 0]
        a = arr[:, 1] if shape == "va" else full
    if color == 3:
        s8 = np.uint64(bits - 8)
        code = (r >> s8) | (g >> s8) << np.uint64(8) | (b >> s8) << np.uint64(16) | (a >> s8) << np.uint64(24)
        pal = np.frombuffer(bytes(palette), np.uint8).reshape(-1, 4).astype(np.uint64)
        pcode = pal[:, 0] | pal[:, 1] << np.uint64(8) | pal[:, 2] << np.uint64(16) | pal[:, 3] << np.uint64(24)
        u, first = np.unique(pcode, return_index=True)  # first match wins for duplicate entries
        at = np.minimum(np.searchsorted(u, code), len(u) - 1)
        return np.where(u[at] == code, first[at], 0).astype(np.uint8).tobytes()
    s = {0: (r,), 4: (r, a), 2: (b, g, r) if bgr else (r, g, b), 6: (b, g, r, a) if bgr else (r, g, b, a)}[color]
    out = np.stack([_narrow(x, bits, depth) for x in s], axis=1)
    return out.astype(">u2" if depth == 16 else "u1").tobytes()
