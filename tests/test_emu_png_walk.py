"""png_walk_kernel (csrc/png_walk.cuh), both passes, under the host SIMT emulator at three lane orders: every summary
against the oracle's restatement of decompress(stream:) (status, a, b, header, format, palette) and against the host
walk behind pngb200_png_inspect_batch, and every record list against a plain Python walk of the chunk headers.  The
inputs are the golden fixtures, the structural cases, every fixture cut at and around each chunk boundary and inside a
header, 0xffffffff length fields, and IDAT runs of 1 to 65 equal chunks, plain and broken at the speculative step's
lanes 0, 1, 31 and 32 (a chunk of another length, an invalid type, a non-IDAT chunk, a body past the end)."""
from __future__ import annotations

import ctypes as C
import os
import struct
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import container_cases as cc  # noqa: E402
import emu  # noqa: E402
import pngio  # noqa: E402
from conftest import GOLDEN  # noqa: E402

SHUFFLED = 5
NONE = (1 << 64) - 1


class Rec(C.Structure):
    _fields_ = [("off", C.c_uint64), ("len", C.c_uint32), ("type", C.c_uint32), ("declared", C.c_uint32)]


def summary_type(pkg):
    class Head(C.Structure):
        _fields_ = [("status", C.c_int32), ("a", C.c_uint32), ("b", C.c_uint32), ("stop_before_crc", C.c_uint32),
                    ("stop", C.c_uint64), ("first_idat", C.c_uint64), ("idat_end", C.c_uint64), ("chunks", C.c_uint64),
                    ("width", C.c_uint32), ("height", C.c_uint32), ("depth", C.c_uint8), ("color", C.c_uint8),
                    ("interlaced", C.c_uint8), ("standard", C.c_uint8), ("idat_chunks", C.c_uint32),
                    ("format", pkg.PixelFormat), ("storage_size", C.c_uint64), ("idat_bytes", C.c_uint64),
                    ("palette_entries", C.c_uint32), ("pad", C.c_uint32)]

    class Summary(C.Structure):
        _fields_ = [("head", Head), ("palette_rgba", C.c_uint8 * 1024)]

    return Summary


def run(pkg, files, order):
    L = emu.load("emu_png_walk")
    L.emu_walk_summary_size.restype = C.c_size_t
    L.emu_chunk_rec_size.restype = C.c_size_t
    Summary = summary_type(pkg)
    assert L.emu_walk_summary_size() == C.sizeof(Summary) and L.emu_chunk_rec_size() == C.sizeof(Rec)
    n = len(files)
    bufs = [(C.c_uint8 * max(len(f), 1)).from_buffer_copy(f or b"\0") for f in files]
    ptrs = (C.c_void_p * n)(*[C.addressof(b) if f else None for b, f in zip(bufs, files)])
    lens = (C.c_uint64 * n)(*[len(f) for f in files])
    sums = (Summary * n)()
    cap = sum(max(0, (len(f) - 8) // 12) for f in files) + 1
    recs = (Rec * cap)()
    L.emu_png_walk.restype = C.c_longlong
    L.emu_png_walk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
    total = L.emu_png_walk(n, ptrs, lens, sums, recs, cap, order)
    assert total >= 0
    out, at = [], 0
    for s in sums:
        k = s.head.chunks
        out.append((s, [(r.off, r.len, r.type, r.declared) for r in recs[at: at + k]]))
        at += k
    assert at == total
    return out


def python_records(data: bytes):
    """every chunk header that lexes, from the signature on, as (off, len, type, declared)"""
    out, at = [], 8
    while len(data) - at >= 8:
        n, t = struct.unpack_from(">II", data, at)
        if len(data) - at - 8 < n + 4:
            break
        out.append((at, n, t, struct.unpack_from(">I", data, at + 8 + n)[0]))
        at += 12 + n
    return out if data[:8] == pngio.SIGNATURE else []


def idat_run(recs):
    first = next((k for k, r in enumerate(recs) if r[2] == cc.fourcc("IDAT")), None)
    if first is None:
        return 0, 0
    k = first
    while k < len(recs) and recs[k][2] == cc.fourcc("IDAT"):
        k += 1
    return k - first, sum(r[1] for r in recs[first:k])


def check(pkg, orc, files, order):
    got = run(pkg, files, order)
    host = pkg.png_inspect(files)
    for data, (s, recs), im in zip(files, got, host):
        h = s.head
        why = (data[:48], h.status, order)
        # the host adapter: every field pngb200_png_inspect_batch fills
        assert (h.status, h.a, h.b, h.chunks, h.idat_chunks, h.idat_bytes) == \
               (im.status, im.err_a, im.err_b, im.chunks, im.idat_chunks, im.idat_bytes), why
        assert (h.width, h.height, h.depth, h.color, bool(h.interlaced), h.standard) == \
               (im.width, im.height, im.depth, im.color, im.interlaced, im.standard), why
        f = h.format
        fields = dict(color=f.color, depth=f.depth, bgr=bool(f.bgr),
                      key=tuple(f.key[: 1 if f.color == 0 else 3]) if f.has_key else None,
                      palette=bytes(s.palette_rgba[: 4 * f.palette_count]) if f.color == 3 else None)
        assert fields == im.fields, why
        # the oracle (its CRC check aside: that runs on the device behind the walk)
        info = orc.png_inspect(data)
        if info.status != orc.ERR_LEX_INVALID_CHUNK_CHECKSUM:
            assert (h.status, h.a, h.b) == (info.status, info.a, info.b), why
            if info.status == 0:
                assert (h.width, h.height, h.depth, h.color, h.interlaced, h.standard) == \
                       (info.width, info.height, info.depth, info.color, info.interlaced, info.standard), why
                assert fields == info.fields(), why
        # the records: a prefix of the plain header walk, and the IDAT run they describe
        want = python_records(data)
        assert recs == want[: len(recs)], why
        if h.first_idat == NONE:  # stopped before the first IDAT was accepted
            assert (h.idat_chunks, h.idat_bytes) == (0, 0), why
        else:
            run_chunks, run_bytes = idat_run(recs)
            assert (h.idat_chunks, h.idat_bytes) == (run_chunks, run_bytes), why
            assert recs[h.first_idat][2] == cc.fourcc("IDAT") and h.idat_end - h.first_idat == run_chunks, why
            assert all(r[2] != cc.fourcc("IDAT") for r in recs[: h.first_idat]), why
        if h.status == 0:
            assert h.stop == NONE and recs[-1][2] == cc.fourcc("IEND"), why
        else:
            assert h.stop == len(recs) - (0 if h.stop_before_crc else 1), why


def fixtures():
    out = []
    for sub in ("pngsuite", "ios", "invalid"):
        for f in sorted(os.listdir(os.path.join(GOLDEN, sub))):
            if f.endswith(".png"):
                out.append(open(os.path.join(GOLDEN, sub, f), "rb").read())
    return out


def cuts(data: bytes):
    """the file cut at each chunk boundary -1, 0 and +1, and inside each chunk header"""
    out = set()
    for off, *_ in python_records(data) + [(len(data),)]:
        for at in (off - 1, off, off + 1, off + 5):
            if 0 <= at < len(data):
                out.add(data[:at])
    return sorted(out, key=len)


HEAD = pngio.SIGNATURE + cc.chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 4, 8, 0, 0, 0, 0))
IEND = cc.chunk(b"IEND", b"")


def run_file(lens, breaker=None, at=None, tail=IEND):
    """a grey file whose IDAT run has chunks of `lens` bytes; `breaker` replaces chunk `at` of the run"""
    body = []
    for k, n in enumerate(lens):
        payload = bytes((7 * k + j) & 0xFF for j in range(n))
        body.append(breaker(payload) if k == at and breaker else cc.chunk(b"IDAT", payload))
    return HEAD + b"".join(body) + tail


def runs():
    out = []
    for k in (1, 31, 32, 33, 65):
        out.append(run_file([16] * k))
        out.append(run_file([16] * (k - 1) + [5]))
        out.append(run_file([0] * k))
    breakers = [lambda p: cc.chunk(b"IDAT", p[:-1]),         # another length
                lambda p: cc.chunk(b"ID\x00T", p),            # an invalid type
                lambda p: cc.chunk(b"tEXt", b"k\0" + p)]      # a chunk that is not IDAT
    for lane in (0, 1, 31, 32):
        at = 1 + lane  # the first IDAT is lexed before the warp speculates: lane j looks at run chunk 1 + j
        for b in breakers:
            out.append(run_file([16] * 40, b, at))
            out.append(run_file([16] * 70, b, at))
        whole = run_file([16] * 40)
        cut = 8 + 25 + at * 28 + 8 + 7    # inside the body of run chunk `at`
        out.append(whole[:cut])
        out.append(whole[:cut - 7 + 16 + 2])  # inside its CRC
    out.append(HEAD + struct.pack(">I", 0xFFFFFFFF) + b"IDAT" + bytes(40))
    out.append(run_file([16] * 3, tail=struct.pack(">I", 0xFFFFFFFF) + b"IDAT" + bytes(40)))
    out.append(run_file([16] * 40, tail=struct.pack(">I", 0xFFFFFFFF) + b"tEXt" + bytes(40)))
    out.append(HEAD[:8] + struct.pack(">I", 0xFFFFFFFF) + b"IHDR" + bytes(13))
    return out


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_fixtures_and_structural_cases(pngb200, orc, order):
    files = fixtures() + [d for d, _ in cc.structural_cases(orc)] + [b"", b"\x89PNG\r\n\x1a"]
    check(pngb200, orc, files, order)


@pytest.mark.parametrize("order", [0, 1, SHUFFLED])
def test_idat_runs_and_breaks(pngb200, orc, order):
    check(pngb200, orc, runs(), order)


@pytest.mark.parametrize("order", [0, SHUFFLED])
def test_every_fixture_cut_at_its_chunk_boundaries(pngb200, orc, order):
    files = []
    for data in fixtures() + runs()[:12]:
        files += cuts(data)
    check(pngb200, orc, files, order)
