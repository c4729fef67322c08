"""ctypes binding of tests/deflate_stream.c, the CPU restatement of LZ77.Deflator's streaming behaviour (test
infrastructure only), and the push schedules the online-deflator tests share."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE = os.path.join(HERE, "..", "oracle")
ZLIB, IOS, GZIP = 0, 1, 2
CHUNK = 65544       # 2 x the capacity malloc gives DeflatorOut's 32 768 UInt16 atoms: the default chunk


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "deflate_stream.c")
    lib = os.path.join(HERE, "libdeflate_stream.so")
    deps = [src] + [os.path.join(ORACLE, f) for f in ("lz77_deflate.c", "lz77_inflate.c", "oracle.h")]
    if force or not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["gcc", "-O2", "-std=c11", "-shared", "-fPIC", "-I" + ORACLE, "-o", lib, src,
                        os.path.join(ORACLE, "lz77_inflate.c")], check=True)
    return lib


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_deflator_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t]
        L.orc_deflator_create.restype = C.c_void_p
        L.orc_deflator_destroy.argtypes = [C.c_void_p]
        L.orc_deflator_push.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int]
        for f in (L.orc_deflator_pop, L.orc_deflator_pull):
            f.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
        L.orc_deflator_progress.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


class StreamingDeflator:
    """LZ77.Deflator / Gzip.Deflator push(_:last:), pop(), pull() on the CPU, the shape of the library's online
    Deflator"""

    def __init__(self, fmt: int = ZLIB, level: int = 9, exponent: int = 15, chunk_bytes: int = CHUNK):
        self.handle = lib().orc_deflator_create(fmt, level, exponent, chunk_bytes)
        assert self.handle, "bad format / exponent / chunk"

    def close(self):
        if getattr(self, "handle", None):
            lib().orc_deflator_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, data: bytes, last: bool = False):
        assert lib().orc_deflator_push(self.handle, bytes(data), len(data), int(last)) == 0, "push after last"

    def _take(self, fn):
        p, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        return C.string_at(p, n.value) if fn(self.handle, C.byref(p), C.byref(n)) else None

    def pop(self):
        return self._take(lib().orc_deflator_pop)

    def pull(self):
        return self._take(lib().orc_deflator_pull)

    def progress(self) -> tuple:
        """(input bytes dequeued, complete bytes written including the header, blocks, pending input bytes)"""
        out = (C.c_uint64 * 4)()
        lib().orc_deflator_progress(self.handle, out)
        return tuple(out)


def drain(d, final: bool = False) -> list:
    """pop() until nil, then after the last push pull() until nil: the chunks a caller gets now"""
    out = []
    while (c := d.pop()) is not None:
        out.append(c)
    while final and (c := d.pull()) is not None:
        out.append(c)
    return out


def cuts(n: int, sizes) -> list:
    """[(start, end)] pieces of a stream of n bytes, cycling through `sizes`"""
    out, at, k = [], 0, 0
    while at < n:
        s = sizes[k % len(sizes)]
        out.append((at, min(n, at + s)))
        at += s
        k += 1
    return out
