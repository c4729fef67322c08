"""The streaming inflator's resume point under the host SIMT emulator (tests/emu): inflate_serial_kernel and
inflate_wave_kernel run one launch per push, as pngb200_inflator_push launches them, through a job with a resume
record.  Streams are cut into prefixes, each push resumes where the last one stopped (at a block header, or inside a
Huffman block at the last complete symbol), and after every push the bytes, status and error payload are held to the
oracle's one-shot inflate of the same prefix.  The kernels' work counters must show each input bit decoded about once."""
from __future__ import annotations

import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import deflate_craft as dc  # noqa: E402
import emu  # noqa: E402
from oracle import oracle  # noqa: E402

ZLIB, RAW, GZIP = 0, 1, 2   # pngb200_format: zlib, ios (raw deflate), gzip
WRAP = {ZLIB: "zlib", RAW: "raw", GZIP: "gzip"}
HEAD = {ZLIB: 2, RAW: 0, GZIP: 10}   # wrapper header bytes in front of the blocks
NEED_MORE = 1
SERIAL, WAVE, HOST = 0, 1, 2         # HOST: the ring kernel from 64 KiB of undecoded input on, as the handle chooses
ORDERS = [0, 1, 5]                   # lane orders: ascending, descending, a seeded shuffle


class Resume(C.Structure):
    _fields_ = [("header_bit", C.c_uint64), ("symbol_bit", C.c_uint64), ("out", C.c_uint64), ("final", C.c_uint32),
                ("pad", C.c_uint32), ("bits", C.c_uint64), ("bytes", C.c_uint64), ("serial_bytes", C.c_uint64)]


@pytest.fixture(scope="module")
def lib():
    L = emu.load("emu_inflate_resume")
    assert L.emu_result_size() == C.sizeof(emu.Result)
    assert L.emu_resume_size() == C.sizeof(Resume)
    L.emu_inflate_resume.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_uint64,
                                     C.c_uint64, C.c_int, C.POINTER(Resume), C.POINTER(emu.Result), C.c_int]
    L.emu_wave_bits.restype = C.c_uint32
    return L


class Handle:
    """pngb200_inflator_push's state and launch loop over one stream (the whole stream sits in `src`; a push of the
    first n bytes hands the kernel a source of n bytes)"""

    def __init__(self, L, stream: bytes, cap: int, fmt: int, engine: int, order: int):
        self.L, self.fmt, self.engine, self.order = L, fmt, engine, order
        self.src = (C.c_uint8 * (len(stream) + 16)).from_buffer_copy(stream + bytes(16))
        self.cap = cap
        self.dst = (C.c_uint8 * (cap + 64))()
        self.at = Resume()
        self.bit = self.out = self.phase = 0
        self.status, self.err, self.produced = NEED_MORE, (0, 0), 0
        self.steps = []   # per launch: (engine, bits, bytes, serial_bytes, start bit, prefix bytes)

    def push(self, n: int):
        if self.status != NEED_MORE:
            return
        pending = n - min(n, self.bit >> 3)
        eng = self.engine if self.engine != HOST else (WAVE if pending >= 64 << 10 else SERIAL)
        r = emu.Result()
        start = self.bit
        self.L.emu_inflate_resume(eng, C.addressof(self.src), n, C.addressof(self.dst), self.cap, self.fmt, self.bit,
                                  self.out, self.phase, C.byref(self.at), C.byref(r), self.order)
        self.steps.append((eng, self.at.bits, self.at.bytes, self.at.serial_bytes, start, n))
        self.bit, self.out, self.phase = r.resume_bit, r.resume_out, r.phase
        self.status, self.err, self.produced = r.status, (r.err_a, r.err_b), r.produced
        if r.phase == 3:
            assert (self.at.symbol_bit, self.at.out) == (r.resume_bit, r.resume_out)
            assert self.at.header_bit < self.at.symbol_bit

    def output(self) -> bytes:
        return bytes(self.dst)[:self.produced]

    def work(self):
        return tuple(sum(s[k] for s in self.steps) for k in (1, 2, 3))


def stored_spans(blocks, end_bit):
    """(header bit, end bit, output offset) of every stored block (Writer.finish's stream-relative block list)"""
    spans = []
    for k, (b, o, t) in enumerate(blocks):
        if t == 0:
            spans.append((b, blocks[k + 1][0] if k + 1 < len(blocks) else end_bit, o))
    return spans


def expect(stream: bytes, n: int, fmt: int, cap: int, spans):
    """the oracle's inflate of the first n bytes, with the handle's one difference: a stored block is released once
    all of it has arrived"""
    st, out, res = oracle.inflate(stream[:n], fmt, cap)
    if st == NEED_MORE:
        for b0, b1, o in spans:
            if b0 < 8 * n < b1:
                out = out[:o]
    return st, out, (res.a, res.b)


def run_cuts(L, case_or_stream, fmt, cuts, engine=HOST, order=0, check_every=True):
    if isinstance(case_or_stream, dc.Case):
        stream, plain, blocks = case_or_stream.stream(WRAP[fmt])
        spans = stored_spans(blocks, case_or_stream.writer.end_bit + 8 * HEAD[fmt])
    else:
        stream, plain, spans = case_or_stream
    full_st, full, _ = oracle.inflate(stream, fmt)
    cap = max(len(full), 1)
    h = Handle(L, stream, cap, fmt, engine, order)
    for k, n in enumerate(cuts):
        h.push(n)
        if check_every or k == len(cuts) - 1:
            st, out, err = expect(stream, n, fmt, cap, spans)
            assert (h.status, h.produced) == (st, len(out)), (n, h.status, h.produced, st, len(out))
            assert h.output() == out, n
            if st < 0:
                assert h.err == err, (n, h.err, err)
        if h.status != NEED_MORE:
            break
    return h, stream


def cut_points(total: int, step: int, start: int = 0):
    return list(range(start or step, total, step)) + [total]


# ---- where a cut falls: a small DEFLATE reader that records every field boundary ----
class Bits:
    def __init__(self, data: bytes, pos: int = 0):
        self.b = np.unpackbits(np.frombuffer(data, np.uint8), bitorder="little")
        self.pos = pos

    def get(self, n: int) -> int:
        v = int(sum(int(x) << k for k, x in enumerate(self.b[self.pos:self.pos + n])))
        self.pos += n
        return v


def _decoder(lens):
    codes = dc.canonical(lens)
    return {(n, dc.reverse(c, n)): s for s, (c, n) in enumerate(zip(codes, lens)) if n}


def _sym(br: Bits, table) -> int:
    v = 0
    for n in range(1, 16):
        v |= int(br.b[br.pos + n - 1]) << (n - 1)
        if (n, v) in table:
            br.pos += n
            return table[(n, v)]
    raise ValueError("bad code")


def cut_classes(stream: bytes, head: int):
    """{bit: set of classes} for every bit position of a valid stream (classes of the interior of a field are given to
    every bit strictly inside it)"""
    br = Bits(stream, 8 * head)
    cls: dict[int, set] = {}

    def mark(lo, hi, name, inclusive_lo=False):
        for p in range(lo if inclusive_lo else lo + 1, hi):
            cls.setdefault(p, set()).add(name)

    final = False
    while not final:
        h0 = br.pos
        final, btype = br.get(1), br.get(2)
        if btype == 0:
            br.pos = (br.pos + 7) & ~7
            l0 = br.pos
            n = br.get(16)
            br.get(16)
            mark(l0, br.pos, "stored LEN/NLEN")
            mark(br.pos, br.pos + 8 * n, "stored payload", inclusive_lo=n > 0)
            br.pos += 8 * n
            end = br.pos
        else:
            if btype == 1:
                lit, dist = _decoder(dc.FIXED_LIT), _decoder(dc.FIXED_DIST)
            else:
                hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[dc.CL_ORDER[i]] = br.get(3)
                ct = _decoder(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = _sym(br, ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.get(2))
                    else:
                        lens += [0] * ((3 + br.get(3)) if s == 17 else (11 + br.get(7)))
                lit, dist = _decoder(lens[:hlit]), _decoder(lens[hlit:])
                mark(h0, br.pos, "dynamic header")
            while True:
                t0 = br.pos
                cls.setdefault(t0, set()).add("symbol boundary")
                s = _sym(br, lit)
                if s < 256:
                    mark(t0, br.pos, "literal code")
                elif s == 256:
                    mark(t0, br.pos, "inside EOB")
                    cls.setdefault(br.pos, set()).add("just after EOB")
                    break
                else:
                    e = dc.LEN_EXTRA[s - 257]
                    if e:
                        cls.setdefault(br.pos, set()).add("between length code and extra bits")
                    br.pos += e
                    cls.setdefault(br.pos, set()).add("between length and distance")
                    ds = _sym(br, dist)
                    e = dc.DIST_EXTRA[ds]
                    if e:
                        mark(br.pos, br.pos + e, "inside distance extra bits")
                    br.pos += e
            end = br.pos
    trailer = (end + 7) & ~7
    for p in range(end, trailer + 1):   # the final block's end, up to the byte boundary the trailer starts at
        cls.setdefault(p, set()).add("final block end")
    mark(trailer, 8 * len(stream), "inside trailer", inclusive_lo=True)
    return cls


def small_stream(seed: int = 3):
    """a few KiB holding every field a cut can fall into: stored, fixed and dynamic blocks, every length and distance
    symbol with its extra bits, empty blocks"""
    rng = np.random.default_rng(seed)
    w = dc.Writer()
    w.stored(rng.integers(0, 256, 300, dtype=np.uint8).tobytes())
    tokens = [rng.integers(0, 256, 200, dtype=np.uint8).tobytes()]
    for k in range(29):
        for n in (dc.LEN_BASE[k], dc.LEN_BASE[k] + (1 << dc.LEN_EXTRA[k]) - 1):
            tokens += [(n, int(rng.integers(1, 500))), int(rng.integers(0, 256))]
    w.fixed(tokens)
    dc._phase(w, 0)   # a block whose EOB ends on a byte boundary
    w.fixed([])
    tokens = [rng.integers(0, 256, 400, dtype=np.uint8).tobytes()]
    for dk in range(30):
        d = dc.DIST_BASE[dk] + int(rng.integers(0, 1 << dc.DIST_EXTRA[dk]))
        if d <= 1500:
            tokens += [(int(rng.integers(3, 259)), d), int(rng.integers(0, 256))]
    tokens += [(int(rng.integers(3, 259)), int(rng.integers(1, 1000))) for _ in range(200)]
    w.dynamic(tokens, *dc._freq_lengths(tokens))
    w.stored(b"")
    tokens = [rng.integers(0, 256, 300, dtype=np.uint8).tobytes(), (100, 700), (7, 3)]
    w.dynamic(tokens, *dc._freq_lengths(tokens), final=True)
    return dc.Case("small", w)


@pytest.mark.parametrize("fmt,order", [(ZLIB, 0), (ZLIB, 1), (ZLIB, 5), (GZIP, 0), (RAW, 0)])
def test_one_byte_pushes_small_stream(lib, fmt, order):
    """every byte offset of a small stream is a cut, so the cuts fall into every field: inside a literal code, between
    a length code and its extra bits, between length and distance, inside the distance extra bits, on a symbol
    boundary, inside and just after EOB, inside a dynamic header, stored LEN/NLEN and payload, the final block's end
    and the trailer"""
    case = small_stream()
    stream, _, _ = case.stream(WRAP[fmt])
    h, _ = run_cuts(lib, case, fmt, list(range(1, len(stream) + 1)), engine=SERIAL, order=order)
    assert h.status == 0
    cls = cut_classes(stream, HEAD[fmt])
    seen = set().union(*(cls.get(8 * n, set()) for n in range(1, len(stream) + 1)))
    want = {"literal code", "between length code and extra bits", "between length and distance",
            "inside distance extra bits", "symbol boundary", "inside EOB", "dynamic header", "stored LEN/NLEN",
            "stored payload", "just after EOB", "final block end"} | ({"inside trailer"} if fmt != RAW else set())
    assert want <= seen, want - seen
    # each byte is decoded once; the dynamic header of the block in flight is parsed again on every push
    bits, nbytes, serial = h.work()
    assert nbytes == len(h.output()) == serial
    assert bits <= 8 * len(stream) + len(stream) * 600


@pytest.mark.parametrize("name", ["fixed_long", "far_window", "sparse_trees", "header_straddle", "empty_blocks"])
@pytest.mark.parametrize("fmt", [ZLIB, GZIP, RAW])
def test_craft_families(lib, name, fmt):
    """pushes of uneven sizes, below and above the ring kernel's 64 KiB: both kernels resume each other's points"""
    case = dc.build(name, 150_000, seed=1)
    stream, _, _ = case.stream(WRAP[fmt])
    rng = np.random.default_rng(len(stream))
    cuts, n = [], 0
    while n < len(stream):
        n = min(len(stream), n + int(rng.choice([7, 1000, 9000, 70_000, 90_000])))
        cuts.append(n)
    h, _ = run_cuts(lib, case, fmt, cuts, order=5 if fmt == ZLIB else 0)
    assert h.status == 0


@pytest.mark.parametrize("name", sorted(dc.INVALID))
def test_defects_in_a_later_push(lib, name):
    """the defect lies after several resume points; every push before it and the one that meets it match the oracle"""
    case = dc.build(name, 40_000, seed=2)
    stream, _, _ = case.stream("zlib")
    h, _ = run_cuts(lib, case, ZLIB, cut_points(len(stream), len(stream) // 7 + 1), engine=SERIAL)
    assert (h.status, h.err) == (case.status, case.err)
    assert len(h.steps) > 5


@pytest.mark.parametrize("name", ["bad_hdist31_used", "bad_fixed_lit286", "bad_distance_past_start", "bad_lit_incomplete"])
def test_defects_through_the_ring_kernel(lib, name):
    """a push that meets the defect in the ring kernel falls back from the last wave checkpoint: same status and
    payload as the oracle"""
    case = dc.build(name, 200_000, seed=2)
    stream, _, _ = case.stream("zlib")
    h, _ = run_cuts(lib, case, ZLIB, cut_points(len(stream), 70_001), engine=WAVE)
    assert (h.status, h.err) == (case.status, case.err)


def test_zlib_level9(lib):
    rng = np.random.default_rng(9)
    base = rng.integers(0, 256, 4000, dtype=np.uint8).tobytes()
    plain = b"".join(base[int(rng.integers(0, 3000)):][:int(rng.integers(50, 900))] for _ in range(400))
    z = zlib.compress(plain, 9)
    h, _ = run_cuts(lib, (z, plain, []), ZLIB, cut_points(len(z), 977))
    assert h.status == 0 and h.output() == plain


def one_big_block(seed: int = 4):
    """a single dynamic block of more than 1 MiB of output"""
    rng = np.random.default_rng(seed)
    w = dc.Writer()
    base = rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes()
    tokens = [base]
    while sum(len(t) if isinstance(t, bytes) else t[0] for t in tokens) < (1 << 20) + 100_000:
        tokens.append(rng.integers(0, 256, int(rng.integers(20, 120)), dtype=np.uint8).tobytes())
        tokens.append((int(rng.integers(3, 259)), int(rng.integers(1, 32769))))
    w.dynamic(tokens, *dc._freq_lengths(tokens), final=True)
    return dc.Case("one_big_block", w)


@pytest.mark.parametrize("order", [0, 5])
def test_ring_kernel_hands_the_serial_decoder_at_most_one_wave(lib, order):
    case = one_big_block()
    stream, plain, blocks = case.stream("zlib")
    assert len(blocks) == 1 and len(plain) > 1 << 20
    WV_BITS = lib.emu_wave_bits()
    cuts = cut_points(len(stream), 64 << 10)
    h, _ = run_cuts(lib, case, ZLIB, cuts, engine=WAVE, order=order)
    assert h.status == 0 and h.output() == plain
    br = Bits(stream, 16 + 3)
    hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
    header_bits = 3 + 14 + 3 * hclen + 2 * (hlit + hdist) * 7   # an upper bound on the header's length
    for eng, bits, nbytes, serial, start, n in h.steps:
        assert eng == WAVE
        # the serial decoder starts at the last wave checkpoint, less than one wave (+ the token that crosses its end)
        # before the end of the input
        lo = max(0, (8 * n - WV_BITS - 64) // 8)
        lo_out = len(oracle.inflate(stream[:lo], ZLIB, len(plain))[1])
        hi_out = len(oracle.inflate(stream[:n], ZLIB, len(plain))[1]) if n < len(stream) else len(plain)
        assert serial <= hi_out - lo_out, (n, serial, hi_out - lo_out)
    bits, nbytes, serial = h.work()
    assert bits <= 8 * len(stream) + len(h.steps) * (header_bits + WV_BITS)
    assert nbytes == len(plain)
