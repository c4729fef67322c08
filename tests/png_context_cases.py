"""Shared pieces of the online-decoding tests (PNG.Context): golden files with their IDAT chunks, streams whose filtered
bytes arrive at chosen offsets, and an independent model of PNG.Image.assign + PNG.Image.overdraw."""
from __future__ import annotations

import ctypes as C
import os
import struct
import zlib

import numpy as np

import pngio
from oracle import oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ADAM7 = ((0, 0, 3, 3), (4, 0, 3, 3), (0, 4, 2, 3), (2, 0, 2, 2), (0, 2, 1, 2), (1, 0, 1, 1), (0, 1, 0, 1))


def goldens():
    """(name, file bytes) of every PngSuite, ios and colour golden"""
    out = []
    for sub in ("pngsuite", "ios", "colour"):
        d = os.path.join(GOLDEN, sub)
        out += [(f"{sub}/{n}", open(os.path.join(d, n), "rb").read()) for n in sorted(os.listdir(d)) if n.endswith(".png")]
    return out


def geometry(png):
    """keyword arguments of a context for a parsed file"""
    return dict(w=png.width, h=png.height, volume=png.volume, depth=png.depth, interlaced=png.interlaced,
                standard=png.fmt)


def passes(w, h, interlaced):
    """[(z, bx, by, ex, ey, width, height)] of the non-empty passes"""
    if not interlaced:
        return [(0, 0, 0, 0, 0, w, h)]
    out = []
    for z, (bx, by, ex, ey) in enumerate(ADAM7):
        pw, ph = (w + (1 << ex) - bx - 1) >> ex, (h + (1 << ey) - by - 1) >> ey
        if pw > 0 and ph > 0:
            out.append((z, bx, by, ex, ey, pw, ph))
    return out


def row_ends(w, h, volume, interlaced):
    """[(z, r, end)]: row r of pass z is complete once `end` filtered bytes are available"""
    out, at = [], 0
    for z, bx, by, ex, ey, pw, ph in passes(w, h, interlaced):
        pitch = (pw * volume + 7) >> 3
        for r in range(ph):
            at += pitch + 1
            out.append((z, r, at))
    return out


def none_stream(storage, w, h, volume, depth, interlaced):
    """the filtered stream of an image with every row's filter byte None: each row is its own reconstruction"""
    bpp = (volume + 7) >> 3
    px = np.frombuffer(storage, np.uint8).reshape(h, w, bpp)
    out = bytearray()
    for z, bx, by, ex, ey, pw, ph in passes(w, h, interlaced):
        pitch = (pw * volume + 7) >> 3
        for r in range(ph):
            row = px[by + (r << ey), bx::1 << ex][:pw]
            line = bytearray(pitch)
            if depth < 8:
                per = 8 // depth
                for i, v in enumerate(row[:, 0]):
                    line[i // per] |= (int(v) & ((1 << depth) - 1)) << ((per - 1 - i % per) * depth)
            else:
                line[:] = row.tobytes()
            out += b"\x00" + line
    return bytes(out)


def stored_zlib(data: bytes, block: int = 1000) -> bytes:
    """a zlib stream of stored blocks of `block` bytes: the reference's inflator releases their bytes as they arrive"""
    out = bytearray(b"\x78\x01")
    for i in range(0, max(len(data), 1), block):
        piece = data[i:i + block]
        out += bytes([1 if i + block >= len(data) else 0]) + struct.pack("<HH", len(piece), len(piece) ^ 0xFFFF) + piece
    return bytes(out + struct.pack(">I", zlib.adler32(data)))


def stored_prefix(n: int, block: int = 1000) -> int:
    """bytes of stored_zlib(data, block) to push for exactly the first n data bytes to be available"""
    return 2 + n + 5 * ((n + block - 1) // block)


def random_storage(w, h, volume, depth, seed):
    rng = np.random.default_rng(seed)
    bpp = (volume + 7) >> 3
    px = rng.integers(0, 256, w * h * bpp, dtype=np.uint8)
    if depth < 8:
        px &= (1 << depth) - 1
    return px.tobytes()


class OverdrawModel:
    """PNG.Context.push(data:overdraw:)'s delegate, restated in Python from the reference (PNG.Context.swift:89-95,
    PNG.Image.swift:133-183): assign the row, then paint its brush"""

    def __init__(self, w, h, volume, interlaced, final):
        self.w, self.h, self.bpp, self.interlaced = w, h, (volume + 7) >> 3, interlaced
        self.final = np.frombuffer(final, np.uint8).reshape(h, w, self.bpp)
        self.img = np.zeros_like(self.final)

    def row(self, z, r, overdraw):
        bx, by, ex, ey = ADAM7[z] if self.interlaced else (0, 0, 0, 0)
        y = by + (r << ey)
        self.img[y, bx::1 << ex] = self.final[y, bx::1 << ex]
        if not overdraw:
            return
        brx, bry = (1 << ex) >> (bx != 0), (1 << ey) >> (y & 7 != 0)
        if brx * bry <= 1:
            return
        for yy in range(y, min(y + bry, self.h)):
            for x in range(bx, self.w, brx):
                self.img[yy, x:min(x + brx, self.w)] = self.img[y, x]

    def storage(self) -> bytes:
        return self.img.tobytes()


def _orc():
    """liboracle.so with the argument types of oracle/png_context.c's entry points"""
    L = oracle.lib()
    if not getattr(L, "_png_context_bound", False):
        L.orc_png_context_create.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc_png_context_create.restype = C.c_void_p
        L.orc_png_context_push.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int]
        L.orc_png_context_push.restype = C.c_int
        L.orc_png_context_end.argtypes = [C.c_void_p]
        L.orc_png_context_end.restype = C.c_int
        L.orc_png_context_progress.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.orc_png_context_progress.restype = None
        L.orc_png_context_storage.argtypes = [C.c_void_p]
        L.orc_png_context_storage.restype = C.c_void_p
        L.orc_png_context_error.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32),
                                            C.POINTER(C.c_uint32)]
        L.orc_png_context_error.restype = None
        L.orc_png_context_destroy.argtypes = [C.c_void_p]
        L.orc_png_context_destroy.restype = None
        L._png_context_bound = True
    return L


class OracleContext:
    """The oracle's PNG.Context (oracle/png_context.c) with uninitialized: false: push(data, overdraw) -> status,
    end() -> status, progress() -> six values, storage() -> bytes, error() -> (status, a, b)."""

    def __init__(self, w: int, h: int, volume: int, depth: int, interlaced: bool = False, standard: int = 0):
        self._lib = _orc()
        self._size = oracle.storage_size(w, h, volume)
        self.handle = self._lib.orc_png_context_create(w, h, volume, depth, int(interlaced), standard)

    def close(self):
        if getattr(self, "handle", None):
            self._lib.orc_png_context_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, data: bytes, overdraw: bool = False) -> int:
        return self._lib.orc_png_context_push(self.handle, bytes(data), len(data), int(overdraw))

    def end(self) -> int:
        return self._lib.orc_png_context_end(self.handle)

    def progress(self):
        out = (C.c_uint64 * 6)()
        self._lib.orc_png_context_progress(self.handle, out)
        return tuple(out)

    def storage(self) -> bytes:
        return C.string_at(self._lib.orc_png_context_storage(self.handle), self._size)

    def error(self):
        s, a, b = C.c_int(), C.c_uint32(), C.c_uint32()
        self._lib.orc_png_context_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
        return s.value, a.value, b.value
