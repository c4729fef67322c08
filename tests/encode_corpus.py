"""Seeded encoder edge corpus for deflate_kernel (csrc/deflate.cuh), and `blocks`, a small DEFLATE reader that says which
edges a compressed stream really reaches.

Each family builds its cases at two sizes: "emu" (small enough for the SIMT emulator in the CPU suite) and "gpu".
A Case carries a `reach(stats, level, exponent)` check, run on the stream the oracle writes for it: it asserts that
the case still hits the edge it exists for (a 2^e - 1 distance, a 2047-term block, a 15-bit code cut by the length
limiter...), so a corpus that drifts off its edge fails instead of passing without testing anything.

The parse rules the families aim at (DeflatorSearch.init(level:) as deflate_kernel restates it): levels <= 3 parse
greedily, 4..7 lazily, both in blocks of at most 2047 terms (lazy stops its main loop at one free slot); levels >= 8
("full") minimise over a graph of every position, in blocks of 2047, 4095, 8191 ... vertices up to DF_GRAPH_CAP = 2^21,
and walk the dictionary 32 positions at a time.  Levels <= 0 behave as 0, levels >= 13 as 13."""
from __future__ import annotations

import heapq
import zlib
from collections import Counter
from dataclasses import dataclass
from typing import Callable

import numpy as np

import corpus
from deflate_craft import CL_ORDER, DIST_BASE, DIST_EXTRA, LEN_BASE, LEN_EXTRA

ZLIB, IOS, GZIP = 0, 1, 2      # pngb200.FORMAT_* and oracle.ZLIB / IOS / GZIP
DF_GRAPH_CAP = 1 << 21


def mode(level: int) -> int:
    """0 greedy, 1 lazy, 2 full"""
    return 0 if level <= 3 else 1 if level <= 7 else 2


# ---------------------------------------------------------------------------------------------------------------------
# coverage reader


def _unlimited_depth(freqs) -> int:
    """height of a Huffman tree over the nonzero frequencies, ties merged shallowest first (the lowest optimal tree)"""
    heap = [(f, 0) for f in freqs if f]
    if len(heap) < 2:
        return len(heap)
    heapq.heapify(heap)
    while len(heap) > 1:
        fa, da = heapq.heappop(heap)
        fb, db = heapq.heappop(heap)
        heapq.heappush(heap, (fa + fb, max(da, db) + 1))
    return heap[0][1]


class _Bits:
    def __init__(self, data: bytes):
        self.data = data
        self.pos = 0
        self.end = 8 * len(data)

    def peek(self, n: int) -> int:
        """the next n <= 32 bits, LSB first; bits past the end read as zeros"""
        at = self.pos >> 3
        return (int.from_bytes(self.data[at:at + 5], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def get(self, n: int) -> int:
        if self.pos + n > self.end:
            raise ValueError("truncated stream")
        r = self.peek(n)
        self.pos += n
        return r


def _table(lens):
    """LSB-first lookup table of a canonical code: index = next `width` bits -> (symbol, length)"""
    width = max(lens)
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    table = [None] * (1 << width)
    for s, n in enumerate(lens):
        if not n:
            continue
        c = nxt[n]
        nxt[n] += 1
        r = int(f"{c:0{n}b}"[::-1], 2)
        for hi in range(1 << (width - n)):
            table[r | hi << n] = (s, n)
    return table, width


def _decode(bits: _Bits, tw):
    table, width = tw
    e = table[bits.peek(width)]
    if e is None:
        raise ValueError("bad code")
    bits.pos += e[1]
    if bits.pos > bits.end:
        raise ValueError("truncated stream")
    return e[0]


def strip(stream: bytes, fmt: int) -> bytes:
    """the raw DEFLATE data inside a zlib / gzip / raw (.ios) stream"""
    if fmt == ZLIB:
        return stream[2:]
    if fmt == GZIP:
        return stream[10:]
    return stream


def blocks(stream: bytes, fmt: int = ZLIB):
    """(per-block stats, decoded bytes) of a stream.  Per block: type, final, hlit, hdist, hclen, ll_max (longest
    literal/length code), cl_max (longest code-length code), ll_free / cl_free (the height an unlimited Huffman tree
    over the block's used symbols would have), terms (literals + copies, end-of-block not counted), copies, out (bytes
    decoded), max_dist, n258 and pairs (Counter of (length, distance))."""
    bits = _Bits(strip(stream, fmt))
    out = bytearray()
    stats = []
    while True:
        final, btype = bits.get(1), bits.get(2)
        b = dict(type=btype, final=final, hlit=0, hdist=0, hclen=0, ll_max=0, cl_max=0, ll_free=0, cl_free=0, terms=0,
                 copies=0, out=0, max_dist=0, n258=0, pairs=Counter())
        start = len(out)
        if btype == 0:
            bits.pos = (bits.pos + 7) & ~7
            n, nn = bits.get(16), bits.get(16)
            assert n == nn ^ 0xFFFF
            for _ in range(n):
                out.append(bits.get(8))
        elif btype in (1, 2):
            if btype == 1:
                ll = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
                dl = [5] * 30
            else:
                hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                cll = [0] * 19
                for i in range(hclen):
                    cll[CL_ORDER[i]] = bits.get(3)
                ct = _table(cll)
                seq, used = [], Counter()
                while len(seq) < hlit + hdist:
                    s = _decode(bits, ct)
                    used[s] += 1
                    if s < 16:
                        seq.append(s)
                    elif s == 16:
                        seq += [seq[-1]] * (3 + bits.get(2))
                    elif s == 17:
                        seq += [0] * (3 + bits.get(3))
                    else:
                        seq += [0] * (11 + bits.get(7))
                assert len(seq) == hlit + hdist
                ll, dl = seq[:hlit], seq[hlit:]
                b.update(hlit=hlit, hdist=hdist, hclen=hclen, cl_max=max(cll), cl_free=_unlimited_depth(used.values()))
            b["ll_max"] = max(ll)
            lt = _table(ll)
            dt = _table(dl) if max(dl) else None
            freq = Counter()
            while True:
                s = _decode(bits, lt)
                freq[s] += 1
                if s < 256:
                    out.append(s)
                    b["terms"] += 1
                elif s == 256:
                    break
                else:
                    k = s - 257
                    n = LEN_BASE[k] + bits.get(LEN_EXTRA[k])
                    dc = _decode(bits, dt)
                    d = DIST_BASE[dc] + bits.get(DIST_EXTRA[dc])
                    assert 0 < d <= len(out)
                    for _ in range(n):
                        out.append(out[-d])
                    b["terms"] += 1
                    b["copies"] += 1
                    b["max_dist"] = max(b["max_dist"], d)
                    b["n258"] += n == 258
                    b["pairs"][(n, d)] += 1
            b["ll_free"] = _unlimited_depth(freq.values())
        else:
            raise ValueError("block type 3")
        b["out"] = len(out) - start
        stats.append(b)
        if final:
            return stats, bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# the families


@dataclass
class Case:
    family: str
    name: str
    data: bytes
    reach: Callable[[list, int, int], None] | None = None   # (block stats, level, exponent) -> asserts the edge


def check_reach(case: Case, stream: bytes, fmt: int, level: int, exponent: int):
    """decode the stream with the reader, compare with zlib and the input, then run the case's own edge check"""
    stats, plain = blocks(stream, fmt)
    assert plain == case.data, case.name
    wbits = {ZLIB: 15, GZIP: 31, IOS: -15}[fmt]
    assert zlib.decompress(stream, wbits) == case.data, case.name
    if case.reach is not None:
        case.reach(stats, level, 15 if fmt == IOS else exponent)
    return stats


def _rng(tag: str, seed: int):
    return np.random.default_rng([seed, zlib.crc32(tag.encode())])


def _noise(rng, n: int) -> bytes:
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def literal_blocks(n: int, level: int):
    """terms per block of an input the parse takes as all literals (greedy / lazy)"""
    sizes, count = [], 0
    for i in range(n):
        lazy_main = mode(level) == 1 and i < n - 3
        if 2047 - count <= (1 if lazy_main else 0):
            sizes.append(count)
            count = 0
        count += 1
    return sizes + [count]


def full_blocks(n: int):
    """vertices (= bytes) per block of full mode: 2047, 4095, 8191 ... up to the graph cap"""
    sizes, limit = [], 2048
    while n > limit - 1:
        sizes.append(limit - 1)
        n -= limit - 1
        limit = min(2 * limit, DF_GRAPH_CAP)
    return sizes + [n]


def tiny(size: str, seed: int = 1):
    """n = 0 .. 8 (stored path below 3, compress path from 3), 1-, 2- and 3-byte inputs over every byte value"""
    rng = _rng("tiny", seed)
    cases = [Case("tiny", f"count{n}", bytes(rng.integers(0, 256, n, dtype=np.uint8))) for n in range(9)]
    cases += [Case("tiny", f"zeros{n}", bytes(n)) for n in (1, 2, 3, 4, 7, 8, 300)]

    def stored(stats, level, exponent):
        assert len(stats) == 1 and stats[0]["type"] == 0

    for width in (1, 2, 3):
        for v in range(256):
            data = bytes((v + 37 * k) & 0xFF for k in range(width))
            cases.append(Case("tiny", f"w{width}v{v}", data, stored if width < 3 else None))
    for c in cases[:3]:
        c.reach = stored
    return cases


def window(size: str, seed: int = 1):
    """a random motif that recurs at a period of 2^e - 1, 2^e and 2^e + 1 with random filler between: at exponent e the
    first copy sits at distance `mask` (the longest the window allows), the others must not be used"""
    exps = (8, 9, 12) if size == "emu" else (8, 12, 15)
    rng = _rng("window", seed)
    cases = []
    for e in exps:
        for period in ((1 << e) - 1, 1 << e, (1 << e) + 1):
            m = min(300, period // 2)
            motif = _noise(rng, m)
            data = b"".join(motif + _noise(rng, period - m) for _ in range(2)) + motif

            def reach(stats, level, exponent, e=e, period=period):
                far = max(b["max_dist"] for b in stats)
                used = {d for b in stats for (_, d) in b["pairs"]}
                if exponent == e:
                    assert far == period if period == (1 << e) - 1 else far < (1 << e) - 1, (far, period)
                elif period < (1 << exponent) - 1:
                    assert period in used, (far, period)
            cases.append(Case("window", f"e{e}p{period}", data, reach))
    return cases


def _kernel_hash(k: int) -> int:
    return ((k * 2654435761) & 0xFFFFFFFF) >> 16


def colliding_keys(rng, groups: int, per: int = 3):
    """`groups` sets of `per` distinct 4-byte keys with one kernel hash each, by brute force over seeded keys"""
    keys = rng.integers(0, 1 << 32, 1 << 18, dtype=np.uint64)
    h = ((keys * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(16)
    by = {}
    for k, hv in zip(keys.tolist(), h.tolist()):
        s = by.setdefault(hv, set())
        s.add(k)
    found = [sorted(s)[:per] for s in by.values() if len(s) >= per]
    assert len(found) >= groups
    return found[:groups]


def batch_collisions(data: bytes, limit: int) -> int:
    """32-position batches (aligned to the stream start, as in a first full-mode block) holding at least two distinct
    keys with one hash and one key seen twice"""
    hits = 0
    for a0 in range(0, min(len(data) - 3, limit) - 31, 32):
        keys = [int.from_bytes(data[a0 + i:a0 + i + 4], "big") for i in range(32)]
        by = {}
        for k in keys:
            by.setdefault(_kernel_hash(k), set()).add(k)
        shared_hash = any(len(s) >= 2 for s in by.values())
        repeated_key = len(set(keys)) < 32
        hits += shared_hash and repeated_key
    return hits


def hash_collisions(size: str, seed: int = 1):
    """keys that share the kernel's dictionary hash but not their bytes, several inside one 32-position batch, the
    same key twice in a batch; the chunks recur so the hash chains hold the other keys of the bucket"""
    rng = _rng("hash", seed)
    groups = colliding_keys(rng, 8)
    chunks = 60 if size == "emu" else 400
    out = bytearray()
    for j in range(chunks):
        g = groups[(j * 5 + j // 8) % len(groups)]
        k1, k2, k3 = (x.to_bytes(4, "big") for x in g)
        order = [k1, k2, k3, k1] if j % 3 else [k3, k1, k2, k3]
        body = b"".join(order)
        out += body + _noise(rng, 32 - len(body)) if j % 4 else body + body[:16]
    data = bytes(out)

    def reach(stats, level, exponent):
        assert sum(b["copies"] for b in stats) > 0
    assert batch_collisions(data, 2016) >= 40
    return [Case("hash", "buckets", data, reach)]


def long_runs(size: str, seed: int = 1):
    """runs of 258, 259, 358 and more bytes crossing 32-position batch edges (full mode skips the vertices after a
    match longer than 100), copies of exactly 258 bytes, and a long run across the first block's vertex limit"""
    rng = _rng("runs", seed)
    cases = []
    out = bytearray()
    for i, run in enumerate((258, 259, 358, 600, 1000)):
        out += _noise(rng, 17 + 7 * i) + bytes([i + 1]) * run
    cases.append(Case("runs", "runs", bytes(out)))
    blockr = _noise(rng, 258)
    copies = _noise(rng, 21) + blockr + _noise(rng, 40) + blockr + _noise(rng, 77) + blockr + _noise(rng, 30)
    cases.append(Case("runs", "copy258", copies))
    cases.append(Case("runs", "edge", _noise(rng, 1990) + bytes(420) + _noise(rng, 300)))

    def reach(stats, level, exponent):
        assert sum(b["n258"] for b in stats) >= 1

    def copy(stats, level, exponent):   # a 258-byte copy of noise lies 298 bytes back: beyond an exponent-8 window
        assert sum(b["n258"] for b in stats) >= (1 if exponent > 8 else 0)
    cases[0].reach, cases[1].reach = reach, copy

    def edge(stats, level, exponent):   # full mode: the run is cut at 2047 vertices and both blocks copy from it
        if mode(level) == 2:
            assert stats[0]["out"] == 2047
            assert all(any(d == 1 and n > 50 for (n, d) in b["pairs"]) for b in stats[:2])
        else:
            assert sum(b["n258"] for b in stats) >= 1
    cases[2].reach = edge
    return cases


def lazy_choice(size: str, seed: int = 1):
    """the match at a + 1 longer than, as long as, and shorter than the one at a: the lazy parse defers only when it is
    strictly longer (er < lr)"""
    rng = _rng("lazy", seed)
    cases = []
    for name, er, lr in (("longer", 12, 16), ("equal", 20, 20), ("shorter", 30, 25)):
        r = _noise(rng, 48)
        tail = max(er, lr + 1) + 3
        seg_a = r[:er] + bytes([r[er] ^ 0x55])           # r[0:er], then a byte that ends the match
        seg_b = r[1:1 + lr] + bytes([r[1 + lr] ^ 0x55])   # r[1:1 + lr], likewise
        at_a = 40
        at_b = at_a + len(seg_a) + 33
        copy_at = at_b + len(seg_b) + 29
        data = _noise(rng, 40) + seg_a + _noise(rng, 33) + seg_b + _noise(rng, 29) + r[:tail] + bytes([r[tail] ^ 0x55])
        data += _noise(rng, 50)
        dist_a, dist_b = copy_at - at_a, copy_at + 1 - at_b

        def reach(stats, level, exponent, er=er, lr=lr, dist_a=dist_a, dist_b=dist_b, name=name):
            pairs = sum((b["pairs"] for b in stats), Counter())
            if mode(level) == 1 and name == "longer":
                assert pairs[(lr, dist_b)] == 1 and pairs[(er, dist_a)] == 0, pairs
            elif mode(level) < 2:
                assert pairs[(er, dist_a)] == 1 and pairs[(lr, dist_b)] == 0, pairs
        cases.append(Case("lazy", name, data, reach))
    return cases


def block_edges(size: str, seed: int = 1):
    """all-literal noise of 2046, 2047, 2048 and 4094 terms (greedy / lazy block limits), and compressible inputs
    around the full-mode block ends at 2047, 6142 (2047 + 4095) and 14333 vertices"""
    rng = _rng("blocks", seed)
    cases = []
    for n in (2046, 2047, 2048, 4094):
        def reach(stats, level, exponent, n=n):
            if mode(level) < 2:
                assert [b["terms"] for b in stats] == literal_blocks(n, level)
                assert sum(b["copies"] for b in stats) == 0
            else:
                assert [b["out"] for b in stats] == full_blocks(n)
        cases.append(Case("blocks", f"noise{n}", _noise(rng, n), reach))
    img = corpus.make("graphic", 128, 128, 11).reshape(128, -1)
    text = corpus.filter_rows_numpy(img, 4)
    for n in ((2047, 2048, 6142, 6143) if size == "emu" else (2047, 2048, 6142, 6143, 14333, 14334)):
        def reach(stats, level, exponent, n=n):
            if mode(level) == 2:
                assert [b["out"] for b in stats] == full_blocks(n)
            assert sum(b["copies"] for b in stats) > 0
        cases.append(Case("blocks", f"graphic{n}", text[:n], reach))
    return cases


def skewed(size: str, seed: int = 1):
    """skewed literal frequencies, so that limitHeight has to cut a tree: Zipf-distributed bytes make the code-length
    tree deeper than 7; 32 even symbols plus a tail with Fibonacci counts (1, 1, 2, 3, 5 ...) in the third full-mode
    block (8191 vertices, after 2047 + 4095) make the literal/length tree deeper than 15.  The symbols are random
    enough that the parse keeps them as literals."""
    rng = _rng("skew", seed)
    p = 1.0 / np.arange(1, 257) ** 1.2
    perm = rng.permutation(256).astype(np.uint8)
    zipf = perm[rng.choice(256, size=6000 if size == "emu" else 60000, p=p / p.sum())].tobytes()

    def cl_cut(stats, level, exponent):
        assert any(b["cl_free"] > 7 and b["cl_max"] == 7 for b in stats), [(b["cl_free"], b["cl_max"]) for b in stats]

    # third block: the end-of-block symbol (weight 1) and 11 tail symbols weighing 1, 2, 3, 5 ... 144 form a chain of
    # Huffman merges, 32 bulk symbols share the rest; no 4-byte key recurs anywhere, so the parse has nothing to match
    # and the block's literal frequencies are exactly these counts
    fib = [1, 2]
    while len(fib) < 11:
        fib.append(fib[-1] + fib[-2])
    bulk = list(range(0, 256, 8))
    left = 8191 - sum(fib)
    third = [s + 3 for s, f in zip(bulk, fib) for _ in range(f)]
    third += [bulk[i] for i in range(32) for _ in range(left // 32 + (i < left % 32))]
    head = 2047 + 4095
    pool = [bulk[i] for i in rng.integers(0, 32, head)] + [third[i] for i in rng.permutation(len(third))]
    seen = set()
    for i in range(3, len(pool)):
        while tuple(pool[i - 3:i + 1]) in seen:   # a recurring key: redraw (head) or swap with a later symbol (third)
            if i < head:
                pool[i] = bulk[int(rng.integers(32))]
            else:
                j = int(rng.integers(i, len(pool)))
                pool[i], pool[j] = pool[j], pool[i]
        seen.add(tuple(pool[i - 3:i + 1]))
    fibtail = bytes(pool)

    def ll_cut(stats, level, exponent):
        if mode(level) == 2:
            assert [b["out"] for b in stats][:2] == [2047, 4095]
            assert any(b["ll_free"] > 15 and b["ll_max"] == 15 for b in stats), [(b["ll_free"], b["ll_max"]) for b in stats]
    return [Case("skew", "zipf", zipf, cl_cut), Case("skew", "fibtail", fibtail, ll_cut)]


def png_rows(size: str, seed: int = 1):
    """filtered scanlines of photos and graphics, as the PNG encoder feeds them"""
    w, h = (40, 30) if size == "emu" else (320, 240)
    cases = []
    for kind, idx in (("photo", 3), ("graphic", 4)):
        img = corpus.make(kind, w, h, idx).reshape(h, -1)
        cases.append(Case("png", kind, corpus.filter_rows_numpy(img, 4)))
    img16 = corpus.make("photo", w // 2, h // 2, 6, sixteen=True).reshape(h // 2, -1)
    cases.append(Case("png", "photo16", corpus.filter_rows_numpy(img16, 8)))
    return cases


FAMILIES = {"tiny": tiny, "window": window, "hash": hash_collisions, "runs": long_runs, "lazy": lazy_choice,
            "blocks": block_edges, "skew": skewed, "png": png_rows}


def build(family: str, size: str = "emu", seed: int = 1):
    return FAMILIES[family](size, seed)
