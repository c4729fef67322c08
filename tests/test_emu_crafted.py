"""The crafted DEFLATE corpus (tests/deflate_craft.py) through the whole-stream wave engines, the segment pipeline and the
split head + tail under the host SIMT emulator (tests/emu), against the oracle: the window's far edge (distances 32 767
and 32 768), one-code and empty distance trees, repeats across the literal/distance boundary, 15-bit codes, thousands of
empty blocks, stored blocks at every bit phase, headers at every offset, and header defects that each engine must report
exactly as the reference does (itself or through the serial kernel)."""
from __future__ import annotations

import ctypes as C
import functools
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import deflate_craft as dc  # noqa: E402
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

ZLIB, RAW = 0, 1
SIZE = 90_000            # output bytes of a valid case (the emulator decodes some 100 KB/s per engine)
BAD_PREFIX = 20_000      # valid output in front of an invalid case's defect
ENGINES = {"wave": ("emu_inflate_wave", "emu_inflate_wave"), "cells": ("emu_inflate_cells", "emu_inflate_cells"),
           "parallel": ("emu_inflate_old", "emu_inflate_parallel")}
ARGS = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(emu.Result), C.c_int]


@functools.lru_cache(maxsize=None)
def engine(name):
    lib, fn = ENGINES[name]
    f = getattr(emu.load(lib), fn)
    f.argtypes = ARGS
    return f


@functools.lru_cache(maxsize=None)
def case(name, size, seed=3):
    return dc.build(name, size, seed)


def run(name, z: bytes, cap: int, fmt: int = ZLIB, order: int = 0, misalign: int = 0):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64 + misalign))()
    r = emu.Result()
    st = engine(name)(C.addressof(src), len(z), C.addressof(out) + misalign, cap, fmt, C.byref(r), order)
    return st, bytes(out)[misalign:misalign + r.produced], r


def check_valid(eng, c: dc.Case, wrapper="zlib", order=0, misalign=0):
    z, plain, blocks = c.stream(wrapper)
    fmt = ZLIB if wrapper == "zlib" else RAW
    ost, oout, ores = oracle.inflate(z, oracle.ZLIB if fmt == ZLIB else oracle.IOS, len(plain))
    assert ost == 0 and oout == plain
    st, got, r = run(eng, z, len(plain), fmt, order, misalign)
    assert (st, r.err_a, r.err_b) == (0, 0, 0)
    assert got == plain
    assert (r.blocks, r.consumed_bits) == (ores.blocks, ores.consumed_bits) == (len(blocks), ores.consumed_bits)
    if fmt == ZLIB:
        assert r.checksum == ores.checksum
    assert r.stat[3] == 0, "the engine handed a valid stream to the serial kernel"


@pytest.mark.parametrize("eng", sorted(ENGINES))
@pytest.mark.parametrize("name", sorted(dc.CASES))
def test_valid_families(eng, name):
    """two scheduling orders, output aligned and misaligned by an odd byte count"""
    c = case(name, SIZE)
    check_valid(eng, c, order=0, misalign=0)
    check_valid(eng, c, order=3, misalign=7)


@pytest.mark.parametrize("eng", sorted(ENGINES))
def test_raw_far_window(eng):
    check_valid(eng, case("far_window", SIZE), wrapper="raw", order=1, misalign=3)


@pytest.mark.parametrize("eng", sorted(ENGINES))
@pytest.mark.parametrize("name", sorted(dc.INVALID))
def test_invalid_families(eng, name):
    """the defect sits behind BAD_PREFIX bytes of valid blocks: status and payload are the reference's, whoever decodes"""
    c = case(name, BAD_PREFIX)
    z, plain, _ = c.stream("zlib")
    ost, _, ores = oracle.inflate(z, oracle.ZLIB, len(plain) + 4096)
    assert (ost, ores.a, ores.b) == (c.status, *c.err)
    st, _, r = run(eng, z, len(plain) + 4096)
    assert (st, r.err_a, r.err_b) == (c.status, *c.err)


# ---- segments: block search, symbolic segments, window propagation, marker resolve ----
@functools.lru_cache(maxsize=None)
def seglib():
    L = emu.load("emu_inflate_segments")
    L.emu_inflate_segmented.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    return L


def run_segmented(z: bytes, plain_len: int, nseg: int, plant: int = 0):
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (plain_len + 64))()
    prod, used = C.c_uint64(), C.c_uint32()
    rc = seglib().emu_inflate_segmented(C.addressof(src), len(z), C.addressof(out), plain_len, ZLIB, nseg, plant,
                                        C.byref(prod), C.byref(used))
    return rc, bytes(out)[: prod.value], used.value


@pytest.mark.parametrize("name", sorted(n for n in dc.CASES if dc.build(n, 1, 0).split_points))
def test_segments(name):
    """every family with split points, cut where the block search finds headers"""
    c = case(name, SIZE)
    z, plain, _ = c.stream("zlib")
    rc, got, used = run_segmented(z, len(plain), 3)
    assert rc == 0 and got == plain
    assert used >= 2, "no split point found: the segments were not exercised"


def far_tail(head_len: int, marker_bytes: int, clean: int):
    """a head of random literals, then -- at a planted split point -- a tail whose first copies reach exactly 32 768
    bytes back into the head (`marker_bytes` of them) followed by `clean` literal bytes in the same block, then a stored
    block and a final dynamic block.  Returns (stream, plain, the tail's first bit)."""
    import numpy as np
    rng = np.random.default_rng(17)
    w = dc.Writer()
    head = [rng.integers(0, 256, head_len, dtype=np.uint8).tobytes(), (258, 32768), (258, 1)]
    w.dynamic(head, *dc._freq_lengths(head))
    at = w.bw.pos
    copies, left = [], marker_bytes
    while left:
        n = min(258, left) if left - min(258, left) == 0 or left - min(258, left) >= 3 else left - 3
        copies.append((n, 32768))
        left -= n
    tail = copies + [rng.integers(0, 256, clean, dtype=np.uint8).tobytes()]
    w.dynamic(tail, *dc._freq_lengths(tail))
    w.stored(rng.integers(0, 256, 5_000, dtype=np.uint8).tobytes())
    last = [rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes(), (258, 32768), (100, 32767)]
    w.dynamic(last, *dc._freq_lengths(last), final=True)
    z, plain, _ = w.finish("zlib")
    return z, plain, at + 16


@functools.lru_cache(maxsize=None)
def splitlib():
    L = emu.load("emu_inflate_switch")
    assert L.emu_switch_result_size() == C.sizeof(emu.Result)
    L.emu_inflate_switch.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.c_uint64,
                                     C.c_uint32, C.POINTER(emu.Result), C.POINTER(C.c_uint64), C.POINTER(emu.Result * 2),
                                     C.POINTER(C.c_uint64 * 2)]
    S = emu.load("emu_inflate_split")
    S.emu_inflate_split.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_double, C.c_uint64, C.c_uint64,
                                    C.POINTER(emu.Result), C.POINTER(C.c_uint64), C.POINTER(emu.Result * 2)]
    return L, S


def run_switch(z: bytes, cap: int, plant: int, may_switch: int = 1):
    L, _ = splitlib()
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64))()
    r, at, pieces, sw = emu.Result(), C.c_uint64(), (emu.Result * 2)(), (C.c_uint64 * 2)()
    rc = L.emu_inflate_switch(C.addressof(src), len(z), C.addressof(out), cap, 0.5, plant, 0, may_switch,
                              C.byref(r), C.byref(at), C.byref(pieces), C.byref(sw))
    return rc, bytes(out)[: r.produced], r, pieces, sw[0]


def run_split(z: bytes, cap: int, plant: int):
    _, S = splitlib()
    src = (C.c_uint8 * (len(z) + 8)).from_buffer_copy(z + b"\0" * 8)
    out = (C.c_uint8 * (cap + 64))()
    r, at, pieces = emu.Result(), C.c_uint64(), (emu.Result * 2)()
    rc = S.emu_inflate_split(C.addressof(src), len(z), C.addressof(out), cap, 0.5, plant, 0, C.byref(r), C.byref(at),
                             C.byref(pieces))
    return rc, bytes(out)[: r.produced], r


def same_as_oracle(z, plain, r):
    ost, oout, ores = oracle.inflate(z, oracle.ZLIB, len(plain))
    assert ost == 0 and oout == plain
    assert (r.status, r.checksum, r.blocks, r.produced, r.consumed_bits) == \
           (0, ores.checksum, ores.blocks, len(plain), ores.consumed_bits)


@pytest.mark.parametrize("clean_after", [32768, 32767])
def test_split_tail_reaches_32768_back_and_switches_where_markers_die(clean_after):
    """the tail's first byte is head byte n1 - 32768 (split_resolve_kernel's window index 0); its markers end at M and
    its first block ends at M + clean_after: with 32 768 clean bytes the tail leaves symbolic mode right there, one byte
    fewer and it must not"""
    marker_bytes = 3 * 258 + 100
    z, plain, at = far_tail(40_000, marker_bytes, clean_after)
    rc, got, r, pieces, sw_out = run_switch(z, len(plain), at)
    assert rc == 1 and got == plain
    same_as_oracle(z, plain, r)
    if clean_after == 32768:
        assert sw_out == marker_bytes + 32768
    else:
        assert marker_bytes + 32768 < sw_out < pieces[1].produced
    rc, got, r = run_split(z, len(plain), at)
    assert rc == 1 and got == plain
    same_as_oracle(z, plain, r)
