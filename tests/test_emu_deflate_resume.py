"""deflate_resume_kernel (csrc/deflate.cuh) under the host SIMT emulator against the streaming restatement of
tests/deflate_stream.c: the kernel carries a handle's state across launches, several handles share a launch, and after
every push the complete bytes written so far, the pending input and the blocks must be the oracle's.

EmuHandle drives the kernel as the library's online deflator does (csrc/pngb200_api.cu, deflator_pushes): the input
from the carry's base on, a launch only when more than 4096 bytes are pending or the push is the last, a graph sized for
every vertex the push can add, and the input the kernel slides down when it moves the base."""
from __future__ import annotations

import ctypes as C
import os
import random
import sys

import pytest

import deflate_stream as ds

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

GRAPH_CAP = 1 << 21
DICT_WORDS = (1 << 16) + 2 * 32768
SHUFFLED = 7


class Job(C.Structure):       # DfResumeJob
    _fields_ = [("carry", C.c_void_p), ("inp", C.c_void_p), ("n", C.c_uint64), ("dict", C.c_void_p),
                ("graph", C.c_void_p), ("up", C.c_void_p), ("graph_vertices", C.c_uint64), ("dst", C.c_void_p),
                ("cap", C.c_uint64), ("host_dst", C.c_void_p), ("result", C.c_void_p),
                ("format", C.c_int32), ("level", C.c_int32), ("exponent", C.c_int32), ("last", C.c_int32)]


class Result(C.Structure):    # DfResumeResult
    _fields_ = [("status", C.c_int32), ("blocks", C.c_uint32), ("produced", C.c_uint64), ("base", C.c_uint64),
                ("end_index", C.c_int64), ("count", C.c_int64)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = emu.load("emu_deflate_resume")
        _lib.emu_deflate_carry_size.restype = C.c_size_t
        _lib.emu_deflate_carry_init.argtypes = [C.c_void_p]
        _lib.emu_deflate_resume.argtypes = [C.POINTER(Job), C.c_int, C.c_int]
    return _lib


def header(fmt, exponent):
    if fmt == ds.ZLIB:
        unpaired = (exponent - 8) << 4 | 8
        check = ~(((unpaired << 8) | (unpaired >> 8)) % 31) & 31
        return bytes([unpaired, check])
    return b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" if fmt == ds.GZIP else b""


class EmuHandle:
    def __init__(self, fmt, level, exponent):
        self.fmt, self.level, self.exponent = fmt, level, exponent
        self.full = level >= 8
        self.carry = (C.c_uint8 * lib().emu_deflate_carry_size())()
        lib().emu_deflate_carry_init(self.carry)
        self.dict = (C.c_uint32 * DICT_WORDS)(*([0xCDCDCDCD] * DICT_WORDS))   # device memory is not cleared
        self.graph = (C.c_uint32 * 0)()
        self.live = b""            # input from the base on
        self.total = self.base = self.count = 0
        self.end_index = -3
        self.out = header(fmt, 15 if fmt == ds.IOS else exponent)
        self.blocks = 0

    def pending(self):
        return self.total - max(0, self.base + self.end_index + 3)

    def push(self, data, last):
        """the job of this push, or None when it only enqueues"""
        self.live += data
        self.total += len(data)
        if not (self.pending() > 4096 or last):
            return None
        n = len(self.live)
        if self.full:
            want = min(GRAPH_CAP, self.count + n - self.end_index) + 2
            if want > len(self.graph) // 32:
                g = (C.c_uint32 * (32 * want))()
                C.memmove(g, self.graph, 128 * self.count)
                self.graph = g
        gv = len(self.graph) // 32
        up = (C.c_uint32 * (gv + 1))()
        cap = (self.count if self.full else 8 * self.count) + n - self.end_index   # as the library sizes it
        cap = cap + cap // 2 + 4096 + 4096
        self.inbuf = (C.c_uint8 * (n + 16)).from_buffer_copy(self.live + b"\0" * 16)
        self.dst = (C.c_uint8 * cap)()
        self.host_dst = (C.c_uint8 * cap)()
        self.res = Result()
        self.up = up
        return Job(C.addressof(self.carry), C.addressof(self.inbuf), n, C.addressof(self.dict), C.addressof(self.graph),
                   C.addressof(up), gv, C.addressof(self.dst), cap, C.addressof(self.host_dst), C.addressof(self.res),
                   self.fmt, self.level, self.exponent, int(last))

    def finish(self):
        r = self.res
        assert r.status == 0, r.status
        self.out += bytes(self.host_dst[: r.produced])
        self.blocks += r.blocks
        shift = r.base - self.base
        self.base, self.end_index, self.count = r.base, r.end_index, r.count
        self.live = bytes(self.inbuf[: len(self.live) - shift])   # the kernel slid the input down by the shift
        assert len(self.live) == self.total - self.base
        assert self.base % 32768 == 0


def run(streams, order=0):
    """streams: [(data, level, fmt, exponent, sizes)].  Pushes piece k of every stream in launch k (the handles whose
    push compresses share it), then the last push, checking every handle against its oracle twin after each push."""
    hs = [EmuHandle(fmt, level, exponent) for _, level, fmt, exponent, _ in streams]
    os_ = [ds.StreamingDeflator(fmt, level, exponent, 1) for _, level, fmt, exponent, _ in streams]
    pieces = [ds.cuts(len(s[0]), s[4]) for s in streams]
    seen = [b""] * len(streams)     # the oracle's complete bytes so far (chunks of one byte)
    rounds = max(len(p) for p in pieces) + 1
    for k in range(rounds):
        jobs, live = [], []
        for i, (data, *_rest) in enumerate(streams):
            last = k == len(pieces[i])
            if k > len(pieces[i]):
                continue
            piece = b"" if last else data[pieces[i][k][0]: pieces[i][k][1]]
            os_[i].push(piece, last)
            j = hs[i].push(piece, last)
            if j is not None:
                jobs.append(j)
                live.append(i)
        if jobs:
            arr = (Job * len(jobs))(*jobs)
            lib().emu_deflate_resume(arr, len(jobs), order)
            for i in live:
                hs[i].finish()
        for i in range(len(streams)):
            if k > len(pieces[i]):
                continue
            dequeued, written, blocks, pending = os_[i].progress()
            h = hs[i]
            seen[i] += b"".join(ds.drain(os_[i], k == len(pieces[i])))
            assert len(h.out) == written == len(seen[i]), (i, k, len(h.out), written)
            assert h.out == seen[i], (i, k)
            assert h.blocks == blocks, (i, k, h.blocks, blocks)
            if k < len(pieces[i]):
                assert h.pending() == pending, (i, k, h.pending(), pending)
    for (data, level, fmt, exponent, _), h in zip(streams, hs):
        assert h.out == oracle.deflate(data, level, fmt, exponent), (level, fmt, exponent)
    return hs


def text(n, seed):
    r = random.Random(seed)
    words = [bytes(r.choice(b"abcdefghij") for _ in range(r.randint(2, 9))) for _ in range(60)]
    out = bytearray()
    while len(out) < n:
        out += r.choice(words) + b" "
        if r.random() < 0.02:
            out += bytes(r.getrandbits(8) for _ in range(r.randint(1, 40)))
        if r.random() < 0.01:
            out += bytes([r.getrandbits(8)]) * r.randint(100, 700)   # long matches: the skip rule in full mode
    return bytes(out[:n])


SCHEDULES = {
    "pages": [65544],
    "edges": [4097, 1, 258, 259, 4096, 1, 1, 5000],
    "small": [700, 1300, 3],
    "odd": [4353, 8191, 17],
}


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
@pytest.mark.parametrize("level", [0, 3, 4, 7])
def test_greedy_lazy_every_wrapper(level, order):
    data = text(40000, level)
    run([(data, level, fmt, exp, SCHEDULES[sch])
         for fmt, exp, sch in ((ds.ZLIB, 15, "edges"), (ds.GZIP, 8, "odd"), (ds.IOS, 8, "small"), (ds.ZLIB, 8, "pages"))],
        order)


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
@pytest.mark.parametrize("level", [8, 9])
def test_full_every_wrapper(level, order):
    data = text(24000, 10 + level)
    run([(data, level, fmt, exp, SCHEDULES[sch])
         for fmt, exp, sch in ((ds.ZLIB, 15, "edges"), (ds.GZIP, 8, "odd"), (ds.IOS, 15, "small"))], order)


def test_level13_and_mixed_levels_in_one_launch():
    run([(text(6000, 3), 13, ds.ZLIB, 15, [4097, 1, 1500]),
         (text(30000, 4), 4, ds.GZIP, 15, [4097, 1, 1500]),
         (text(20000, 5), 9, ds.ZLIB, 8, [4097, 1, 1500]),
         (b"ab", 9, ds.GZIP, 15, [1, 1]),
         (b"", 0, ds.ZLIB, 15, [1])], SHUFFLED)


def test_block_limits_and_rebase_over_a_long_stream():
    """greedy blocks of 2048 terms, several base moves of 32 768, exponent 8 and 15 side by side"""
    data = text(200000, 6)
    hs = run([(data, 1, ds.ZLIB, 15, [65544]), (data, 5, ds.ZLIB, 8, [12345])])
    assert all(h.base >= 131072 for h in hs)
