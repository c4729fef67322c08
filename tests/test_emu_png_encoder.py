"""The online encoder's device steps (filter_resume_kernel, deflate_resume_kernel with scanline ends) under the host
SIMT emulator against the restatement of tests/png_encoder_stream.py: several encoders share each launch, and after
every push the filtered scanlines must be oracle.png_filter's bytes and the pieces handed out must be the
restatement's.

EmuEncoder drives the kernels as the library's push call does (csrc/png_file.cuh, encoder_pushes): the scanlines the
rows so far complete, in stream order; a non-interlaced scanline reads the push's rows and a carried copy of the row
before them, an Adam7 one the whole storage received so far (rows not yet pushed are poisoned); the filtered bytes go
onto the end of the deflator's input, whose launch runs only when more than 4096 bytes are pending or the push brings
the last row, with the ends of the push's scanlines.  The pieces are framed here on the host (the CRC-32 kernel is
covered by the GPU tests)."""
from __future__ import annotations

import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import deflate_stream as ds
import png_encoder_stream as pes
import pngio

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

GRAPH_CAP = 1 << 21
DICT_WORDS = (1 << 16) + 2 * 32768
SHUFFLED = 7


class FilterJob(C.Structure):     # FilterResumeJob
    _fields_ = [("rows", C.c_void_p), ("carried", C.c_void_p), ("out", C.c_void_p), ("out_off0", C.c_uint64),
                ("width", C.c_uint32), ("height", C.c_uint32), ("first", C.c_uint32), ("row0", C.c_uint32),
                ("volume", C.c_uint8), ("depth", C.c_uint8), ("interlaced", C.c_uint8), ("bpp", C.c_uint8)]


class Job(C.Structure):           # DfResumeJob
    _fields_ = [("carry", C.c_void_p), ("inp", C.c_void_p), ("n", C.c_uint64), ("dict", C.c_void_p),
                ("graph", C.c_void_p), ("up", C.c_void_p), ("graph_vertices", C.c_uint64), ("dst", C.c_void_p),
                ("cap", C.c_uint64), ("host_dst", C.c_void_p), ("result", C.c_void_p),
                ("format", C.c_int32), ("level", C.c_int32), ("exponent", C.c_int32), ("last", C.c_int32)]


class Ends(C.Structure):          # DfEnds
    _fields_ = [("at", C.c_void_p), ("count", C.c_uint64)]


class Result(C.Structure):        # DfResumeResult
    _fields_ = [("status", C.c_int32), ("blocks", C.c_uint32), ("produced", C.c_uint64), ("base", C.c_uint64),
                ("end_index", C.c_int64), ("count", C.c_int64)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = emu.load("emu_png_encoder")
        _lib.emu_encoder_filter_job_size.restype = C.c_size_t
        _lib.emu_encoder_carry_size.restype = C.c_size_t
        _lib.emu_encoder_carry_init.argtypes = [C.c_void_p]
        _lib.emu_encoder_filter.argtypes = [C.POINTER(FilterJob), C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_int]
        _lib.emu_encoder_deflate.argtypes = [C.POINTER(Job), C.c_int, C.POINTER(Ends), C.c_int]
        assert _lib.emu_encoder_filter_job_size() == C.sizeof(FilterJob)
    return _lib


class EmuEncoder:
    def __init__(self, storage, w, h, fields, interlaced, level, chunk, sched):
        self.storage, self.w, self.h, self.fields, self.interlaced = storage, w, h, fields, interlaced
        self.level, self.chunk, self.sched = level, chunk, sched
        self.vol = pes.volume(fields)
        self.bpp = (self.vol + 7) >> 3
        self.row = w * self.bpp
        self.lines = pes.scanlines(w, h, self.vol, interlaced)
        self.filtered = oracle.png_filter(storage, w, h, self.vol, fields["depth"], interlaced)
        self.want = pes.pieces(oracle, storage, w, h, fields, interlaced, level, chunk, sched)
        self.fmt = ds.IOS if fields.get("bgr") else ds.ZLIB
        self.rows = self.done = self.k = 0
        # Adam7: the storage as received; rows not pushed yet are poisoned, so a read of one shows in the bytes
        self.store = (C.c_uint8 * max(1, len(storage)))(*([0xA5] * len(storage)))
        self.carried = (C.c_uint8 * max(1, self.row))()
        # the online deflator's state, as tests/test_emu_deflate_resume.py keeps it
        self.carry = (C.c_uint8 * lib().emu_encoder_carry_size())()
        lib().emu_encoder_carry_init(self.carry)
        self.dict = (C.c_uint32 * DICT_WORDS)(*([0xCDCDCDCD] * DICT_WORDS))
        self.graph = (C.c_uint32 * 0)()
        self.live, self.total, self.base, self.count, self.end_index = b"", 0, 0, 0, -3
        self.out = b"" if self.fmt == ds.IOS else bytes([0x78, 0x01])   # DeflatorBuffers.init: exponent 15
        self.handed = 0       # payload bytes handed out in chunks

    def offset(self, k):
        return self.lines[k][1] if k < len(self.lines) else len(self.filtered)

    def filter_job(self):
        """the push's rows taken in and its filter job, or None when it completes no scanline"""
        n = self.sched[self.k]
        rows = self.storage[self.rows * self.row: (self.rows + n) * self.row]
        self.push_rows = (C.c_uint8 * max(1, len(rows) + 16)).from_buffer_copy(rows + b"\0" * 16)
        C.memmove(C.addressof(self.store) + self.rows * self.row, self.push_rows, len(rows))
        r1 = self.rows + n
        l1 = self.done
        while l1 < len(self.lines) and self.lines[l1][0] < r1:
            l1 += 1
        self.new = (self.done, l1, r1)
        size = self.offset(l1) - self.offset(self.done)
        self.fout = (C.c_uint8 * max(1, size))()
        if l1 == self.done:
            return None
        return FilterJob(C.addressof(self.store) if self.interlaced else C.addressof(self.push_rows),
                         C.addressof(self.carried), C.addressof(self.fout), self.offset(self.done), self.w, self.h,
                         self.done, self.rows, self.vol, self.fields["depth"], int(self.interlaced), self.bpp)

    def pending(self):
        return self.total - max(0, self.base + self.end_index + 3)

    def deflate_job(self):
        """the filtered bytes counted in; the push's deflate job and ends, or None when it only enqueues"""
        l0, l1, r1 = self.new
        a, b = self.offset(l0), self.offset(l1)
        got = bytes(self.fout[: b - a])
        assert got == self.filtered[a:b], (self.k, l0, l1)
        held = len(self.live)
        self.live += got
        self.total += len(got)
        self.last = r1 == self.h
        if not (self.pending() > 4096 or self.last):
            return None
        n = len(self.live)
        if self.level >= 8:
            want = min(GRAPH_CAP, self.count + n - self.end_index) + 2
            if want > len(self.graph) // 32:
                g = (C.c_uint32 * (32 * want))()
                C.memmove(g, self.graph, 128 * self.count)
                self.graph = g
        gv = len(self.graph) // 32
        self.up = (C.c_uint32 * (gv + 1))()
        cap = (self.count if self.level >= 8 else 8 * self.count) + n - self.end_index
        cap = cap + cap // 2 + 4096 + 4096
        self.inbuf = (C.c_uint8 * (n + 16)).from_buffer_copy(self.live + b"\0" * 16)
        self.dst, self.host_dst, self.res = (C.c_uint8 * cap)(), (C.c_uint8 * cap)(), Result()
        ends = [held + self.offset(k + 1) - a for k in range(l0, l1)]
        self.ends = (C.c_uint64 * max(1, len(ends)))(*ends)
        job = Job(C.addressof(self.carry), C.addressof(self.inbuf), n, C.addressof(self.dict), C.addressof(self.graph),
                  C.addressof(self.up), gv, C.addressof(self.dst), cap, C.addressof(self.host_dst),
                  C.addressof(self.res), self.fmt, self.level, 15, int(self.last))
        return job, Ends(C.addressof(self.ends) if ends else None, len(ends))

    def finish(self, ran):
        """take the launch's result in, move to the next push and check what it hands out"""
        l0, l1, r1 = self.new
        if ran:
            r = self.res
            assert r.status == 0, r.status
            self.out += bytes(self.host_dst[: r.produced])
            shift = r.base - self.base
            self.base, self.end_index, self.count = r.base, r.end_index, r.count
            self.live = bytes(self.inbuf[: len(self.live) - shift])
        if not self.interlaced and r1 > self.rows:
            C.memmove(self.carried, C.addressof(self.push_rows) + (r1 - self.rows - 1) * self.row, self.row)
        got = [self.want[0][0]] if self.k == 0 else []   # the head: built on the host, checked by the GPU tests
        while len(self.out) - self.handed >= self.chunk:
            got.append(pngio.chunk(b"IDAT", self.out[self.handed: self.handed + self.chunk]))
            self.handed += self.chunk
        if r1 == self.h:
            if len(self.out) > self.handed:
                got.append(pngio.chunk(b"IDAT", self.out[self.handed:]))
            got.append(pngio.chunk(b"IEND", b""))
        assert got == self.want[self.k], (self.k, [len(g) for g in got], [len(g) for g in self.want[self.k]])
        self.rows, self.done = r1, l1
        self.k += 1


def run(encoders, order):
    """push k of every encoder in round k: one filter launch and one deflate launch over all of them"""
    for k in range(max(len(e.sched) for e in encoders)):
        live = [e for e in encoders if k < len(e.sched)]
        fjobs, base = [], [0]
        for e in live:
            j = e.filter_job()
            if j is not None:
                fjobs.append(j)
                base.append(base[-1] + e.new[1] - e.new[0])
        if fjobs:
            lib().emu_encoder_filter((FilterJob * len(fjobs))(*fjobs), (C.c_uint32 * len(base))(*base), len(fjobs),
                                     base[-1], order)
        jobs, ends, ran = [], [], []
        for e in live:
            j = e.deflate_job()
            ran.append(j is not None)
            if j is not None:
                jobs.append(j[0])
                ends.append(j[1])
        if jobs:
            lib().emu_encoder_deflate((Job * len(jobs))(*jobs), len(jobs), (Ends * len(ends))(*ends), order)
        for e, r in zip(live, ran):
            e.finish(r)


def noise(fields, w, h, seed):
    rng = np.random.default_rng(seed)
    top = 3 if fields["color"] == 3 else (1 << min(fields["depth"], 8))
    return rng.integers(0, top, w * h * pes.CHANNELS[fields["color"]] * (2 if fields["depth"] == 16 else 1),
                        dtype=np.uint8).tobytes()


def photo(fields, w, h, seed):
    """smooth rows with some noise: compressible, so blocks carry matches"""
    rng = np.random.default_rng(seed)
    n = w * h * pes.CHANNELS[fields["color"]] * (2 if fields["depth"] == 16 else 1)
    x = (np.arange(n) // 7 + rng.integers(0, 3, n)) % 256
    top = 3 if fields["color"] == 3 else (1 << min(fields["depth"], 8))
    return (x % top).astype(np.uint8).tobytes()


PALETTE = bytes([1, 2, 3, 255, 4, 5, 6, 7, 8, 9, 10, 255])
KINDS = (dict(color=6, depth=8), dict(color=0, depth=1), dict(color=0, depth=2, key=(1,)),
         dict(color=3, depth=4, palette=PALETTE), dict(color=2, depth=16, key=(1, 2, 3)),
         dict(color=6, depth=8, bgr=True), dict(color=2, depth=8, bgr=True), dict(color=4, depth=16),
         dict(color=3, depth=2, palette=PALETTE))
LEVELS = (0, 4, 9, 13)


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_adam7_1x1_to_9x9_several_handles_a_launch(order):
    """every Adam7 size from 1x1 to 9x9 (empty passes, one-pixel passes), 1/2/4/8/16-bit and bgr formats, levels
    0/4/9/13, idat_chunk 16, pushes of one row: nine handles in each launch"""
    encs = []
    for s in range(1, 10):
        fields = KINDS[s - 1]
        sched = pes.schedule(s, "rows") if s % 2 else pes.schedule(s, [2, 0, 3])
        encs.append(EmuEncoder(noise(fields, s, s, s), s, s, fields, True, LEVELS[s % 4], 16, sched))
    run(encs, order)


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_formats_levels_and_schedules(order):
    """non-interlaced and Adam7 images of every kind at every level, idat_chunk 16 and 1000, pushes of one row, odd
    bands with empty pushes, and everything at once, all in the same launches"""
    r = random.Random(order)
    encs = []
    for i, fields in enumerate(KINDS):
        w, h = r.randint(3, 40), r.randint(2, 24)
        for interlaced in (False, True):
            kind = ("rows", [3, 0, 5], "all")[(i + interlaced) % 3]
            encs.append(EmuEncoder(photo(fields, w, h, i), w, h, fields, interlaced, LEVELS[(i + interlaced) % 4],
                                   (16, 1000)[i % 2], pes.schedule(h, kind)))
    run(encs, order)


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_scanline_ends_either_side_of_the_trigger(order):
    """scanlines of 4095, 4096 and 4097 filtered bytes: whether a scanline end crosses the 4096-byte trigger decides a
    compression pass, inside a push of many rows as in a push of one (greedy and lazy levels; the full levels run
    scanline ends on the smaller images above)"""
    encs = []
    for w in (4094, 4095, 4096):
        fields = dict(color=0, depth=8)
        px = photo(fields, w, 6, w)
        for level, kind in ((0, "rows"), (4, [2, 3, 1]), (0, "all"), (4, [1, 4, 1])):
            encs.append(EmuEncoder(px, w, 6, fields, False, level, 1000, pes.schedule(6, kind)))
    run(encs, order)
