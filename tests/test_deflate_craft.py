"""The crafted-stream writer (tests/deflate_craft.py) checked against zlib and the oracle: every valid family decodes to
the writer's bytes with the writer's block layout and bit count, every invalid family gets the oracle status and payload
it names, and each family holds the features it exists for."""
from __future__ import annotations

import ctypes as C
import zlib

import pytest

import deflate_craft as dc

SIZE = 120_000
WBITS = {"zlib": 15, "gzip": 31, "raw": -15}


def oracle_fmt(orc, wrapper):
    return {"zlib": orc.ZLIB, "gzip": orc.GZIP, "raw": orc.IOS}[wrapper]


def block_trace(orc, fmt, stream):
    """(bit offset, output offset, BTYPE) of every block the oracle decodes"""
    L = orc.lib()
    L.orc_debug_block_starts.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_size_t]
    L.orc_debug_block_starts.restype = C.c_size_t
    cap = 1 << 15
    trace = (C.c_uint64 * (3 * cap))()
    n = L.orc_debug_block_starts(fmt, stream, len(stream), trace, cap)
    assert n <= cap
    return [(trace[3 * i], trace[3 * i + 1], trace[3 * i + 2]) for i in range(n)]


def test_canonical_codes_and_symbol_tables():
    # RFC 1951 section 3.2.2's example: lengths (3, 3, 3, 3, 3, 2, 4, 4) for A .. H
    assert dc.canonical([3, 3, 3, 3, 3, 2, 4, 4]) == [0b010, 0b011, 0b100, 0b101, 0b110, 0b00, 0b1110, 0b1111]
    assert dc.length_code(3) == (257, 0, 0) and dc.length_code(258) == (285, 0, 0)
    assert dc.length_code(258, alt=True) == (284, 31, 5) and dc.length_code(257) == (284, 30, 5)
    assert dc.dist_code(32768) == (29, 8191, 13) and dc.dist_code(24577) == (29, 0, 13) and dc.dist_code(1) == (0, 0, 0)
    assert dc.kraft(dc.fix_kraft([1, 1, 1, 1])) == 1 << 15
    assert dc.kraft(dc.fix_kraft([15] * 30)) == 1 << 15
    assert dc.kraft(dc.fix_kraft([1, 2, 3, 15, 15, 9], pinned=(0,))) == 1 << 15


@pytest.mark.parametrize("name", sorted(dc.CASES))
@pytest.mark.parametrize("wrapper", ["zlib", "gzip", "raw"])
def test_valid_family_decodes_to_its_bytes(orc, name, wrapper):
    case = dc.build(name, SIZE, seed=1)
    stream, plain, blocks = case.stream(wrapper)
    if case.zlib_agrees:
        assert zlib.decompress(stream, WBITS[wrapper]) == plain
    else:
        # HDIST 31 / 32: zlib refuses the header; the reference accepts it and fails only on a use of symbol 30 / 31,
        # so the oracle (the authority for this project) decodes the stream
        with pytest.raises(zlib.error):
            zlib.decompress(stream, WBITS[wrapper])
    fmt = oracle_fmt(orc, wrapper)
    st, out, res = orc.inflate(stream, fmt, len(plain))
    assert st == 0 and out == plain
    assert res.blocks == len(blocks)
    end = 8 * len(stream) if wrapper != "raw" else case.writer.end_bit
    assert res.consumed_bits == end
    assert block_trace(orc, fmt, stream) == blocks


@pytest.mark.parametrize("name", sorted(dc.INVALID))
def test_invalid_family_gets_its_status(orc, name):
    case = dc.build(name, 40_000, seed=2)
    for wrapper in ("zlib", "raw"):
        stream, plain, blocks = case.stream(wrapper)
        st, _, res = orc.inflate(stream, oracle_fmt(orc, wrapper), len(plain) + 1024)
        assert (st, res.a, res.b) == (case.status, *case.err)
        assert res.blocks == len(blocks) - 1   # the defect is in the last block
        with pytest.raises(zlib.error):        # zlib rejects all of them too (at the header for HDIST 31 / 32)
            zlib.decompress(stream, WBITS[wrapper])


def test_families_hold_what_they_claim():
    seen = {name: dc.build(name, SIZE, seed=1).writer.seen for name in dc.CASES}
    far = seen["far_window"]
    assert {("distance", d) for d in (32767, 32768)} <= far and "15-bit codes" in far and "258 as 284" in far
    assert ("header", 286, 30, 19) in far and ("distance codes", 30) in far
    sparse = seen["sparse_trees"]
    assert ("distance codes", 0) in sparse and ("distance codes", 1) in sparse
    assert ("repeat across", 16) in sparse and (("repeat across", 17) in sparse or ("repeat across", 18) in sparse)
    empty = seen["empty_blocks"]
    assert ("empty", 1) in empty and all(("stored", 0, ph) in empty for ph in range(8))
    assert sum(1 for f in empty if f[0] == "stored" and f[1] == 65535) >= 2
    fixed = seen["fixed_long"]
    assert all(("length symbol", 1, s) in fixed for s in range(257, 286)) and ("distance", 32768) in fixed
    assert "258 as 284" in fixed
    assert ("header", 286, 30, 19) in seen["header_straddle"]
    assert any(f[0] == "header" and f[1:3] == (286, 32) for f in seen["hdist32_unused"])
