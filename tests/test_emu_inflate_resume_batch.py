"""Several streaming inflator pushes in one launch, as pngb200_inflator_push_batch launches them, under the host SIMT
emulator (tests/emu): inflate_serial_kernel with one CTA per job, and inflate_wave_kernel with fewer CTAs than jobs.  The
jobs mix zlib, ios and gzip, resume in phases 0 to 3 (inside fixed and dynamic blocks), and include a job whose output
buffer is too small and a corrupt one.  For every job of every launch the result, the resume record (work counters
included) and the output bytes equal the same job launched alone."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import deflate_craft as dc  # noqa: E402
import emu  # noqa: E402
from oracle import oracle  # noqa: E402
from test_emu_inflate_resume import GZIP, RAW, WRAP, ZLIB, Resume, small_stream  # noqa: E402

NEED_MORE, CAPACITY = 1, -64
SERIAL, WAVE = 0, 1
ORDERS = [0, 1, 5]
FIELDS = ("status", "err_a", "err_b", "checksum", "blocks", "declared", "produced", "consumed_bits", "resume_bit",
          "resume_out", "trailer_seen", "phase", "ck_done")
U64 = C.c_uint64


@pytest.fixture(scope="module")
def lib():
    L = emu.load("emu_inflate_resume_batch")
    L.emu_inflate_resume_batch.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(U64), C.POINTER(C.c_void_p),
                                           C.POINTER(U64), C.POINTER(C.c_int), C.POINTER(U64), C.POINTER(U64),
                                           C.POINTER(C.c_int), C.POINTER(Resume), C.POINTER(emu.Result), C.c_uint, C.c_int]
    return L


class Stream:
    """one handle's state over one stream: the whole stream sits in `src`; a push of the first n bytes hands the kernel
    a source of n bytes"""

    def __init__(self, stream: bytes, fmt: int, cap: int, cuts):
        self.stream, self.fmt, self.cap, self.cuts = stream, fmt, cap, list(cuts)
        self.src = (C.c_uint8 * (len(stream) + 16)).from_buffer_copy(stream + bytes(16))
        self.dst = (C.c_uint8 * (cap + 64))()
        self.at = Resume()
        self.bit = self.out = self.phase = 0
        self.status = NEED_MORE
        self.phases = set()

    def live(self):
        return self.status == NEED_MORE and self.cuts


def launch(L, engine, jobs, grid, order):
    """jobs: [(stream, n, dst buffer, resume record)] in one launch; returns the results"""
    n = len(jobs)
    res = (emu.Result * n)()
    at = (Resume * n)(*[a for _, _, _, a in jobs])
    L.emu_inflate_resume_batch(engine, n, (C.c_void_p * n)(*[C.addressof(s.src) for s, _, _, _ in jobs]),
                               (U64 * n)(*[k for _, k, _, _ in jobs]),
                               (C.c_void_p * n)(*[C.addressof(d) for _, _, d, _ in jobs]),
                               (U64 * n)(*[s.cap for s, _, _, _ in jobs]), (C.c_int * n)(*[s.fmt for s, _, _, _ in jobs]),
                               (U64 * n)(*[s.bit for s, _, _, _ in jobs]), (U64 * n)(*[s.out for s, _, _, _ in jobs]),
                               (C.c_int * n)(*[s.phase for s, _, _, _ in jobs]), at, res, grid, order)
    return list(res), list(at)


def copy_res(a):
    return C.pointer(type(a).from_buffer_copy(a)).contents


def streams():
    """zlib, ios and gzip streams cut at uneven points, a corrupt one and one whose output buffer is too small"""
    out = []
    small = small_stream()
    for fmt in (ZLIB, RAW, GZIP):
        s, _, _ = small.stream(WRAP[fmt])
        out.append(Stream(s, fmt, len(oracle.inflate(s, fmt)[1]), range(13 + 7 * fmt, len(s) + 13 + 7 * fmt, 13 + 7 * fmt)))
    for name, fmt in (("fixed_long", ZLIB), ("sparse_trees", GZIP), ("header_straddle", RAW)):
        s, _, _ = dc.build(name, 30_000, seed=3).stream(WRAP[fmt])
        out.append(Stream(s, fmt, len(oracle.inflate(s, fmt)[1]), range(997, len(s) + 997, 997)))
    bad, _, _ = dc.build("bad_distance_past_start", 30_000, seed=2).stream("zlib")
    out.append(Stream(bad, ZLIB, 1 << 16, range(1500, len(bad) + 1500, 1500)))
    rng = np.random.default_rng(7)
    plain = rng.integers(0, 4, 20_000, dtype=np.uint8).tobytes()
    z = oracle.deflate(plain, 9)
    out.append(Stream(z, ZLIB, 5_000, range(800, len(z) + 800, 800)))   # runs out of output
    for s in out:
        s.cuts = [min(c, len(s.stream)) for c in s.cuts]
    return out


@pytest.mark.parametrize("engine,grid", [(SERIAL, 0), (WAVE, 2)])
@pytest.mark.parametrize("order", ORDERS)
def test_batch_equals_single_launches(lib, engine, grid, order):
    ss = streams()
    launches = 0
    while any(s.live() for s in ss):
        live = [s for s in ss if s.live()]
        jobs, alone = [], []
        for s in live:
            n = s.cuts.pop(0)
            # the job alone, on a copy of the output and the resume record
            d1 = (C.c_uint8 * len(s.dst)).from_buffer_copy(s.dst)
            a1 = Resume.from_buffer_copy(s.at)
            r1, at1 = launch(lib, engine, [(s, n, d1, a1)], max(grid, 1), order)
            alone.append((r1[0], at1[0], bytes(d1)))
            jobs.append((s, n, s.dst, Resume.from_buffer_copy(s.at)))
        res, at = launch(lib, engine, jobs, grid or len(jobs), order)
        launches += 1
        for (s, n, _, _), r, a, (r1, a1, d1) in zip(jobs, res, at, alone):
            assert {f: getattr(r, f) for f in FIELDS} == {f: getattr(r1, f) for f in FIELDS}, (s.fmt, n)
            assert bytes(a) == bytes(a1), (s.fmt, n)
            assert bytes(s.dst) == d1, (s.fmt, n)
            s.phases.add(s.phase)
            s.at = a
            if r.status == CAPACITY:   # the handle grows its output and goes again; here it stops
                s.status = CAPACITY
                continue
            s.bit, s.out, s.phase, s.status = r.resume_bit, r.resume_out, r.phase, r.status
    assert launches > 5
    assert [s.status for s in ss[:6]] == [0] * 6
    assert ss[6].status < 0 and ss[6].status != CAPACITY and ss[7].status == CAPACITY
    assert {0, 1, 3} <= set().union(*(s.phases for s in ss))
