"""deflate_kernel (csrc/deflate.cuh) under the host SIMT emulator against oracle.deflate: every level, window exponent
and wrapper over the encoder edge corpus (tests/encode_corpus.py), under three lane scheduling orders, with warp-slot
reuse, output-capacity errors and the deflate bound.

The emulator runs the kernel on one CTA that takes every job of a batch through its ticket loop (tests/emu/emu_deflate.cpp
says why).  Lane order 0 lets lane 0 run ahead of the other lanes between two warp collectives and order 1 lets it run
last, so a shared-memory word that lane 0 writes while other lanes still read it (or the other way round) gives wrong
bytes here even where the H100 happens to keep the warp converged."""
from __future__ import annotations

import ctypes as C
import os
import sys
import zlib

import pytest

import encode_corpus as ec

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

ERR_OUTPUT_CAPACITY = -64
LEVELS = [-1, 0, 1, 2, 3, 4, 5, 7, 8, 9, 11, 12, 13, 14]
SHUFFLED = 7    # a seeded reshuffle of the lanes every scheduling round


class Job(C.Structure):     # DeflateJob
    _fields_ = [("src", C.c_void_p), ("n", C.c_uint64), ("dst", C.c_void_p), ("cap", C.c_uint64),
                ("format", C.c_int32), ("level", C.c_int32), ("exponent", C.c_int32), ("pad", C.c_int32)]


class Result(C.Structure):  # DeflateResult
    _fields_ = [("status", C.c_int32), ("checksum", C.c_uint32), ("blocks", C.c_uint32), ("pad", C.c_uint32),
                ("produced", C.c_uint64)]


def deflate_bound(n: int) -> int:
    """pngb200_deflate_bound, csrc/pngb200_api.cu: `return n + n / 2 + 4096;`"""
    return n + n // 2 + 4096


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = emu.load("emu_deflate")
        _lib.emu_deflate_batch.argtypes = [C.POINTER(Job), C.c_int, C.POINTER(Result), C.c_int]
    return _lib


def run(specs, order=0, caps=None):
    """specs: [(data, level, fmt, exponent)] -> [(status, bytes written, Result)] from one emulated CTA"""
    n = len(specs)
    jobs, res, keep = (Job * n)(), (Result * n)(), []
    for i, (data, level, fmt, exponent) in enumerate(specs):
        cap = deflate_bound(len(data)) if caps is None else caps[i]
        src = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
        dst = (C.c_uint8 * (cap + 64)).from_buffer_copy(b"\xa5" * (cap + 64))
        keep.append((src, dst, cap))
        jobs[i] = Job(C.addressof(src), len(data), C.addressof(dst), cap, fmt, level, exponent, 0)
    lib().emu_deflate_batch(jobs, n, res, order)
    out = []
    for (src, dst, cap), r in zip(keep, res):
        raw = bytes(dst)
        assert raw[cap:] == b"\xa5" * 64, "written past dst_cap"
        out.append((r.status, raw[:min(r.produced, cap)], r))
    return out


def expect(data, level, fmt, exponent):
    want = oracle.deflate(data, level, fmt, exponent)
    ck = zlib.adler32(data) if fmt == ec.ZLIB else zlib.crc32(data) if fmt == ec.GZIP else 0
    return want, ck


def check(specs, order=0, cases=None):
    got = run(specs, order)
    for i, ((data, level, fmt, exponent), (st, out, r)) in enumerate(zip(specs, got)):
        want, ck = expect(data, level, fmt, exponent)
        tag = (cases[i].name if cases else i, len(data), level, fmt, exponent, order)
        assert st == 0, tag
        assert out == want, tag
        assert r.checksum == ck, tag
        assert r.produced <= deflate_bound(len(data)), tag
        if cases is not None:
            stats = ec.check_reach(cases[i], want, fmt, level, exponent)
            assert r.blocks == len(stats), tag


FMTS = (ec.ZLIB, ec.GZIP, ec.IOS)


def level_slice():
    """(exponent-8 half, exponent-15 half) of a cheap slice of the corpus: full mode at level 13 costs the emulator
    about 2 ms per input byte, so the level sweep keeps to a few KB per level"""
    tiny = [c for c in ec.build("tiny") if c.name.startswith("count") or c.name in ("w1v0", "w2v128", "w3v255", "zeros300")]
    window = [c for c in ec.build("window") if c.name.startswith("e8")]
    runs, lazy = ec.build("runs"), ec.build("lazy")
    return window + ec.build("hash"), tiny + lazy + runs[1:2]


def all_cases():
    return [c for fam in ec.FAMILIES for c in ec.build(fam)]


def window_exponent(case, i):
    """a window case runs at the exponent it is built around, every other case at 8, 9, 12, 15 in turn"""
    return int(case.name[1:case.name.index("p")]) if case.family == "window" else (8, 9, 12, 15)[i % 4]


@pytest.mark.parametrize("level", LEVELS)
def test_every_level_at_exponents_8_and_15(orc, level):
    """a slice of the families at every level (below 0 and above 13 included), one half at exponent 8 and the other at
    15, the three wrappers in turn; one batch per exponent, so the slot runs stream after stream"""
    for exponent, cases in zip((8, 15), level_slice()):
        check([(c.data, level, FMTS[i % 3], exponent) for i, c in enumerate(cases)], 0, cases)


@pytest.mark.parametrize("level", [0, 4, 9])
def test_every_family_at_levels_0_4_9(orc, level):
    """every case of every family at exponents 8, 9, 12 and 15"""
    cases = all_cases()
    check([(c.data, level, FMTS[i % 3], window_exponent(c, i)) for i, c in enumerate(cases)], 0, cases)


@pytest.mark.parametrize("order", [1, SHUFFLED])
@pytest.mark.parametrize("level", [0, 4, 9, 13])
def test_lane_order_does_not_change_the_bytes(orc, order, level):
    """the same streams with lane 0 running last, and with the lanes reshuffled every round"""
    e8, e15 = level_slice()
    cases = e8 + e15 + (ec.build("skew")[:1] if level < 13 else [])
    check([(c.data, level, FMTS[i % 3], window_exponent(c, i)) for i, c in enumerate(cases)], order, cases)


def test_slot_reuse_across_levels_formats_and_exponents(orc):
    """12 streams through one warp slot: its head table is reset per stream, its prevh / next chains and graph are not,
    so an exponent-15 full-mode stream leaves links behind that the exponent-8 streams after it must not follow"""
    w = {c.name: c.data for c in ec.build("window")}
    png = {c.name: c.data for c in ec.build("png")}
    runs = ec.build("runs")[1].data
    specs = [(w["e9p511"], 13, ec.ZLIB, 15), (w["e8p256"], 9, ec.ZLIB, 8), (w["e8p255"], 8, ec.GZIP, 8),
             (png["graphic"][:3000], 11, ec.ZLIB, 15), (w["e8p257"], 12, ec.ZLIB, 8), (runs, 4, ec.GZIP, 8),
             (png["photo"][:2000], 9, ec.IOS, 8), (w["e9p513"], 0, ec.ZLIB, 8), (b"abc", 14, ec.ZLIB, 8),
             (w["e9p512"], 9, ec.ZLIB, 15), (w["e8p255"], 5, ec.ZLIB, 8), (runs, 9, ec.ZLIB, 8)]
    check(specs, 0)


@pytest.mark.parametrize("level", [0, 4, 9])
def test_output_capacity(orc, level):
    """dst_cap 0, 1 and len - 1: ERR_OUTPUT_CAPACITY with the bytes written a prefix of the oracle's and nothing
    written past dst_cap; dst_cap = len: OK"""
    data = ec.build("png")[0].data[:1500]
    for fmt in FMTS:
        want, _ = expect(data, level, fmt, 15)
        caps = [0, 1, len(want) - 1, len(want)]
        got = run([(data, level, fmt, 15)] * 4, 0, caps)
        for cap, (st, out, r) in zip(caps, got):
            if cap < len(want):
                assert st == ERR_OUTPUT_CAPACITY and out == want[:cap], (fmt, cap)
            else:
                assert st == 0 and out == want, (fmt, cap)
            assert r.produced == len(want)    # the writer counts on past the end
