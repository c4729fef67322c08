"""A test-only DEFLATE writer (RFC 1951) for streams that zlib and the reference encoder never write.

zlib and oracle.deflate use a small part of the format: distances up to 32 506 (zlib) or 32 766 (the reference), at
least two distance codes, code lengths sent as two runs, length 258 always as symbol 285.  The writer here takes explicit
code lengths and tokens, so a case can put a copy at distance 32 768, a one-code or empty distance tree, a code-length
repeat across the literal/distance boundary, 15-bit codes, HLIT 286 + HDIST 30 + HCLEN 19 at once, length 258 as
284 + 31, thousands of empty blocks, or one precise header defect.

Writer.finish(wrapper) returns (stream, plain, blocks), `blocks` being (bit offset, output offset, BTYPE) of every block
header in stream bits, as the oracle's block trace reports them.  CASES maps a family name to a seeded builder that
returns a Case at a chosen output size; each invalid family names the oracle status and (err_a, err_b) it must give."""
from __future__ import annotations

import zlib
from dataclasses import dataclass, field

import numpy as np

# ---- RFC 1951 section 3.2.5 ----
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32

# oracle statuses the invalid families expect (oracle/oracle.py)
ERR_RUNLITERAL_SYMBOL_COUNT, ERR_CODELENGTH_HUFFMAN_TABLE, ERR_CODELENGTH_SEQUENCE = -4, -5, -6
ERR_HUFFMAN_TABLE, ERR_STRING_REFERENCE, ERR_INVALID_SYMBOL = -7, -8, -9


def length_code(n: int, alt: bool = False):
    """(symbol, extra value, extra bits) of copy length n; alt: 258 as 284 + 31 instead of 285"""
    if n == 258 and alt:
        return 284, 31, 5
    k = max(i for i, b in enumerate(LEN_BASE) if b <= n)
    return 257 + k, n - LEN_BASE[k], LEN_EXTRA[k]


def dist_code(d: int):
    k = max(i for i, b in enumerate(DIST_BASE) if b <= d)
    return k, d - DIST_BASE[k], DIST_EXTRA[k]


def canonical(lens):
    """canonical Huffman codes (MSB-first values) of code lengths, RFC 1951 section 3.2.2"""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for bits in range(1, 16):
        code = (code + count[bits - 1]) << 1
        nxt[bits] = code
    out = [0] * len(lens)
    for s, n in enumerate(lens):
        if n:
            out[s] = nxt[n]
            nxt[n] += 1
    return out


def reverse(v: int, n: int) -> int:
    return int(f"{v:0{n}b}"[::-1], 2) if n else 0


def kraft(lens, maxlen=15) -> int:
    """sum of 2^(maxlen - l) over the nonzero lengths; 2^maxlen for a complete code"""
    return sum(1 << (maxlen - n) for n in lens if n)


def fix_kraft(lens, maxlen=15, pinned=()):
    """make nonzero lengths a complete prefix code (Kraft sum exactly 1): lengthen the shortest codes while the code is
    over-subscribed, then shorten the codes whose gain fits what is missing, largest gain first (pinned ones stay)"""
    lens = [min(n, maxlen) for n in lens]
    free = sorted((s for s, n in enumerate(lens) if n and s not in pinned), key=lambda s: (lens[s], s))
    count = [0] * (maxlen + 1)
    for s in free:
        count[lens[s]] += 1
    full, k = 1 << maxlen, kraft(lens, maxlen)
    while k > full:
        n = min(n for n in range(1, maxlen) if count[n])
        count[n] -= 1
        count[n + 1] += 1
        k -= 1 << (maxlen - n - 1)
    while k < full:
        n = min(n for n in range(2, maxlen + 1) if count[n] and (1 << (maxlen - n)) <= full - k)
        count[n] -= 1
        count[n - 1] += 1
        k += 1 << (maxlen - n)
    at = 0   # the new lengths, shortest first, in the order of the old ones
    for n in range(1, maxlen + 1):
        for s in free[at:at + count[n]]:
            lens[s] = n
        at += count[n]
    return lens


def huffman_lengths(freqs, maxlen=15):
    """lengths of a complete code over the symbols with nonzero frequency (at least two of them)"""
    import heapq
    used = [s for s, f in enumerate(freqs) if f]
    assert len(used) >= 2
    heap = [(freqs[s], i, [s]) for i, s in enumerate(used)]
    heapq.heapify(heap)
    lens = [0] * len(freqs)
    tie = len(heap)
    while len(heap) > 1:
        fa, _, a = heapq.heappop(heap)
        fb, _, b = heapq.heappop(heap)
        for s in a + b:
            lens[s] += 1
        heapq.heappush(heap, (fa + fb, tie, a + b))
        tie += 1
    return fix_kraft(lens, maxlen)


def random_lengths(n, rng, maxlen=15, lo=1, pinned=None):
    """a complete code over n symbols with random initial lengths in [lo, maxlen] (long codes included)"""
    lens = [int(x) for x in rng.integers(lo, maxlen + 1, n)]
    for s, v in (pinned or {}).items():
        lens[s] = v
    return fix_kraft(lens, maxlen, pinned=tuple(pinned or ()))


class BitWriter:
    """LSB-first bit packer"""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    @property
    def pos(self) -> int:
        return 8 * len(self.out) + self.n

    def put(self, v: int, n: int):
        self.acc |= v << self.n
        self.n += n
        if self.n >= 64:
            k = self.n >> 3
            self.out += (self.acc & ((1 << (8 * k)) - 1)).to_bytes(k, "little")
            self.acc >>= 8 * k
            self.n -= 8 * k

    def put_many(self, vals, lens):
        """a run of codes at once (vals LSB-first, lens <= 32 each)"""
        vals = np.asarray(vals, dtype=np.uint64)
        lens = np.asarray(lens, dtype=np.int64)
        if vals.size == 0:
            return
        width = int(lens.max())
        bits = ((vals[:, None] >> np.arange(width, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8)
        bits = bits[np.arange(width)[None, :] < lens[:, None]]
        pend = np.array([(self.acc >> i) & 1 for i in range(self.n)], dtype=np.uint8)
        allbits = np.concatenate([pend, bits])
        whole = len(allbits) // 8 * 8
        self.out += np.packbits(allbits[:whole], bitorder="little").tobytes()
        rest = allbits[whole:]
        self.acc = sum(int(b) << i for i, b in enumerate(rest))
        self.n = len(rest)

    def align(self):
        if self.n & 7:
            self.put(0, 8 - (self.n & 7))

    def getvalue(self) -> bytes:
        return bytes(self.out) + (self.acc.to_bytes((self.n + 7) // 8, "little") if self.n else b"")


def rle(seq, repeats=True):
    """code-length symbols (sym, extra value, extra bits) for a run of code lengths"""
    out, i = [], 0
    while i < len(seq):
        v, j = seq[i], i
        while j < len(seq) and seq[j] == v:
            j += 1
        run = j - i
        if not repeats:
            out += [(v, 0, 0)] * run
        elif v == 0 and run >= 3:
            while run >= 11:
                k = min(run, 138)
                out.append((18, k - 11, 7))
                run -= k
            if run >= 3:
                out.append((17, run - 3, 3))
                run = 0
            out += [(0, 0, 0)] * run
        else:
            out.append((v, 0, 0))
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, k - 3, 2))
                run -= k
            out += [(v, 0, 0)] * run
        i = j
    return out


class Writer:
    """raw DEFLATE blocks; tokens are a literal byte (int), a literal run (bytes), a copy (length, distance[, alt]),
    ('lsym', s) for a bare literal/length symbol, ('dsym', s) for length 3 with a bare distance symbol, or
    ('draw', value, nbits) for length 3 followed by raw bits where the distance code goes"""

    def __init__(self):
        self.bw = BitWriter()
        self.plain = bytearray()
        self.blocks = []
        self.end_bit = 0
        self.seen = set()   # features written, for the tests that check a family holds what it claims

    def _start(self, btype: int, final: bool):
        self.blocks.append((self.bw.pos, len(self.plain), btype))
        self.bw.put(int(final) | btype << 1, 3)

    def _copy(self, n: int, d: int):
        p = self.plain
        if d >= n:
            p += p[len(p) - d:len(p) - d + n]
        else:
            pat = bytes(p[len(p) - d:])
            p += (pat * (n // d + 1))[:n]

    def _body(self, tokens, lit_lens, dist_lens, btype):
        if not tokens:
            self.seen.add(("empty", btype))
        if 15 in lit_lens:
            self.seen.add("15-bit codes")
        lc = [reverse(c, n) for c, n in zip(canonical(lit_lens), lit_lens)]
        dc = [reverse(c, n) for c, n in zip(canonical(dist_lens), dist_lens)]
        lc_np, ll_np = np.array(lc + [0] * (288 - len(lc)), np.uint64), np.array(list(lit_lens) + [0] * (288 - len(lit_lens)))
        put = self.bw.put
        for t in tokens:
            if isinstance(t, int):
                put(lc[t], lit_lens[t])
                self.plain.append(t)
            elif isinstance(t, (bytes, bytearray)):
                a = np.frombuffer(bytes(t), np.uint8)
                self.bw.put_many(lc_np[a], ll_np[a])
                self.plain += t
            elif t[0] == "lsym":
                put(lc[t[1]], lit_lens[t[1]])
            elif t[0] in ("dsym", "draw"):
                put(lc[257], lit_lens[257])
                if t[0] == "dsym":
                    put(dc[t[1]], dist_lens[t[1]])
                else:
                    put(t[1], t[2])
            else:
                n, d = t[0], t[1]
                s, e, eb = length_code(n, len(t) > 2 and t[2])
                self.seen.add(("length symbol", btype, s))
                if d >= 32767 or (n == 258 and s == 284):
                    self.seen.add(("distance", d) if d >= 32767 else "258 as 284")
                put(lc[s], lit_lens[s])
                put(e, eb)
                k, e, eb = dist_code(d)
                put(dc[k], dist_lens[k])
                put(e, eb)
                self._copy(n, d)
        put(lc[256], lit_lens[256])
        self.end_bit = self.bw.pos

    def stored(self, data: bytes, final: bool = False):
        self.seen.add(("stored", len(data), self.bw.pos % 8))
        self._start(0, final)
        self.bw.align()
        n = len(data)
        self.bw.put(n | (n ^ 0xFFFF) << 16, 32)
        self.bw.out += self.bw.acc.to_bytes(self.bw.n // 8, "little")   # aligned: flush, then the bytes
        self.bw.acc, self.bw.n = 0, 0
        self.bw.out += data
        self.plain += data
        self.end_bit = self.bw.pos

    def fixed(self, tokens, final: bool = False):
        self._start(1, final)
        self._body(tokens, FIXED_LIT, FIXED_DIST, 1)

    def dynamic(self, tokens, lit_lens, dist_lens, final: bool = False, hlit=None, hdist=None, hclen=None,
                runs="split", defect=None):
        """runs: 'none' (every length a symbol), 'split' (two runs, as zlib), 'cross' (one run over both, so repeats
        cross the boundary).  defect: None, 'cl_oversubscribed', 'first_repeat', 'repeat_overrun'."""
        lit_lens, dist_lens = list(lit_lens), list(dist_lens)
        hlit = hlit or max(257, len(lit_lens))
        hdist = hdist or max(1, len(dist_lens))
        lit_lens += [0] * (hlit - len(lit_lens))
        dist_lens += [0] * (hdist - len(dist_lens))
        seq_l, seq_d = lit_lens[:hlit], dist_lens[:hdist]
        if runs == "cross":
            items = rle(seq_l + seq_d)
        else:
            items = rle(seq_l, runs != "none") + rle(seq_d, runs != "none")
        if defect == "first_repeat":
            items = [(16, 0, 2)] + items
        elif defect == "repeat_overrun":
            items = rle(seq_l + seq_d[:-1], runs != "none") + [(18, 127, 7)]
        freqs = [0] * 19
        for s, _, _ in items:
            freqs[s] += 1
        if sum(1 for f in freqs if f) < 2:
            freqs[0 if items[0][0] else 8] += 1
        cl = huffman_lengths(freqs, 7)
        if defect == "cl_oversubscribed":
            cl[next(s for s in CL_ORDER if cl[s] == 0)] = 1
        n_cl = hclen or max(4, max(i + 1 for i, s in enumerate(CL_ORDER) if cl[s]))
        self._start(2, final)
        self.bw.put(hlit - 257, 5)
        self.bw.put(hdist - 1, 5)
        self.bw.put(n_cl - 4, 4)
        for i in range(n_cl):
            self.bw.put(cl[CL_ORDER[i]], 3)
        cc = [reverse(c, n) for c, n in zip(canonical(cl), cl)]
        have = 0
        for s, e, eb in items:
            self.bw.put(cc[s], cl[s])
            self.bw.put(e, eb)
            step = 1 if s < 16 else (3 + e if s < 18 else 11 + e)
            if s >= 16 and have < hlit < have + step:
                self.seen.add(("repeat across", s))
            have += step
        self.seen.add(("header", hlit, hdist, n_cl))
        self.seen.add(("distance codes", sum(1 for n in dist_lens if n)))
        self._body(tokens, lit_lens, dist_lens, 2)

    def finish(self, wrapper: str = "zlib"):
        """(stream, plain, blocks) with a zlib (CINFO 7), gzip or raw wrapper around the blocks"""
        raw, plain = self.bw.getvalue(), bytes(self.plain)
        if wrapper == "raw":
            return raw, plain, list(self.blocks)
        if wrapper == "zlib":
            head, tail = b"\x78\x9c", zlib.adler32(plain).to_bytes(4, "big")
        else:
            head = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff"
            tail = zlib.crc32(plain).to_bytes(4, "little") + (len(plain) & 0xFFFFFFFF).to_bytes(4, "little")
        return head + raw + tail, plain, [(b + 8 * len(head), o, t) for b, o, t in self.blocks]


# ---- case families ----
@dataclass
class Case:
    name: str
    writer: Writer
    status: int = 0                 # oracle status (0: a valid stream)
    err: tuple = (0, 0)             # oracle (err_a, err_b)
    zlib_agrees: bool = True        # zlib decodes it to the same bytes (valid) / rejects it (invalid)
    split_points: bool = True       # holds dynamic headers past the first that block_search takes as split points
    notes: dict = field(default_factory=dict)

    def stream(self, wrapper: str = "zlib"):
        return self.writer.finish(wrapper)

    @property
    def valid(self) -> bool:
        return self.status == 0


def _freq_lengths(tokens, extra_lit=(), extra_dist=(), maxlen=15):
    """code lengths from the tokens' symbol frequencies (every literal of `extra_lit` and EOB included)"""
    fl, fd = [0] * 286, [0] * 30
    fl[256] = 1
    for s in extra_lit:
        fl[s] += 1
    for s in extra_dist:
        fd[s] += 1
    for t in tokens:
        if isinstance(t, int):
            fl[t] += 1
        elif isinstance(t, (bytes, bytearray)):
            for v, c in zip(*np.unique(np.frombuffer(bytes(t), np.uint8), return_counts=True)):
                fl[int(v)] += int(c)
        else:
            fl[length_code(t[0], len(t) > 2 and t[2])[0]] += 1
            fd[dist_code(t[1])[0]] += 1
    if sum(1 for f in fd if f) == 1:
        fd[0 if not fd[0] else 1] += 1
    return huffman_lengths(fl, maxlen), (huffman_lengths(fd, maxlen) if any(fd) else [0])


FAR_DISTANCES = (1, 2, 3, 32506, 32507, 32767, 32768)
FAR_LENGTHS = (3, 4, 100, 257, 258)


def far_window(size: int, seed: int) -> Case:
    """full 286 / 30-symbol trees with random shapes (15-bit codes), HCLEN 19, copies at the window's far edge, blocks
    that open with a copy of distance 32 768"""
    rng = np.random.default_rng(seed)
    w = Writer()
    k = 0
    while len(w.plain) < size:
        # every block after the first opens with a copy from exactly 32 768 bytes back: the first byte of a wave (and
        # of a segment) then comes from the window's first position, s = -32 768
        tokens = [(258, 32768, k % 2 == 1)] if w.plain else []
        tokens += [rng.integers(0, 256, 33_000 if not w.plain else 2_000, dtype=np.uint8).tobytes()]
        for d in FAR_DISTANCES:
            for n in FAR_LENGTHS:
                tokens.append((n, d, n == 258 and (k + d) % 2 == 1))
                tokens.append(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8).tobytes())
        w.dynamic(tokens, random_lengths(286, rng), random_lengths(30, rng), hlit=286, hdist=30, hclen=19,
                  runs=("none", "split", "cross")[k % 3])
        k += 1
    w.fixed([], final=True)
    return Case("far_window", w)


def sparse_trees(size: int, seed: int) -> Case:
    """one-code and empty distance trees, code-length repeats (16, 17, 18) that cross from the literal/length lengths
    into the distance lengths"""
    rng = np.random.default_rng(seed)
    w = Writer()
    w.dynamic([rng.integers(0, 256, 33_000, dtype=np.uint8).tobytes()], *_freq_lengths([bytes(range(256))]))
    k = 0
    while len(w.plain) < size:
        kind = k % 4
        lits = rng.integers(0, 256, 3_000, dtype=np.uint8).tobytes()
        if kind == 0:     # no distance code at all: literals only, HDIST 1 or 5, zeros crossing the boundary
            lit, _ = _freq_lengths([lits])
            w.dynamic([lits], lit, [0] * (1 + 4 * (k % 2)), runs="cross")
        else:             # one distance code of length 1: symbol 0 (distance 1), 3 (4) or 29 (24 577 .. 32 768)
            sym = (0, 3, 29)[kind - 1]
            dists = [1] if sym == 0 else [4] if sym == 3 else [24577, 32768, 30000]
            tokens = [lits] + [(int(rng.integers(3, 259)), int(rng.choice(dists))) for _ in range(60)]
            lit, _ = _freq_lengths(tokens)
            dl = [0] * 30
            dl[sym] = 1
            w.dynamic(tokens, lit, dl[:sym + 1 + (k % 3)], runs="cross")
        k += 1
    # a 16-repeat across the boundary: the last literal/length lengths and the first distance lengths are equal
    tokens = [rng.integers(0, 256, 3_000, dtype=np.uint8).tobytes()] + [(5 + j, 1 + 3 * j) for j in range(40)]
    lit = random_lengths(286, rng, pinned={285: 6, 284: 6, 283: 6})
    dist = random_lengths(30, rng, pinned={0: 6, 1: 6, 2: 6, 3: 6})
    w.dynamic(tokens, lit, dist, hlit=286, hdist=30, runs="cross", final=True)
    return Case("sparse_trees", w)


def _phase(w: Writer, target: int):
    """a fixed block of 9-bit literals that leaves the next block header at bit phase `target`"""
    n9 = (target - w.bw.pos - 10) % 8
    w.fixed([0x90 + j for j in range(n9)])


def empty_blocks(size: int, seed: int) -> Case:
    """thousands of empty fixed and stored blocks between a few with content (7 000 blocks from 1 MiB of output up, 500
    below: the emulator decodes some 130 blocks a second); stored blocks of 0 and 65 535 bytes that start at each of the
    8 bit phases"""
    rng = np.random.default_rng(seed)
    w = Writer()
    w.fixed([rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes()])
    big = min(8, max(2, size // 100_000))
    for ph in range(8):
        _phase(w, ph)
        w.stored(b"")
        if ph < big:
            _phase(w, (ph + 3) % 8)
            w.stored(rng.integers(0, 256, 65_535, dtype=np.uint8).tobytes())
    j = 0
    count = 7000 if size >= 1 << 20 else 500
    while len(w.plain) < size or j < count:
        r = j % 7
        if r in (0, 2, 4):
            w.fixed([])
        elif r in (1, 5):
            w.stored(b"")
        elif r == 3 and j % (count // 10) == 3:
            w.fixed([rng.integers(0, 256, 2_000, dtype=np.uint8).tobytes(), (258, 32768), (258, 1)])
        elif r == 6 and (j % (count // 5) == 6 or j >= count):
            lits = rng.integers(0, 256, 5_000 if j < count else 60_000, dtype=np.uint8).tobytes()
            w.dynamic([lits, (200, 32768)], *_freq_lengths([lits, (200, 32768)]))
        j += 1
    w.stored(b"", final=True)
    return Case("empty_blocks", w)


def fixed_long(size: int, seed: int) -> Case:
    """fixed blocks with every length symbol (280 .. 285 included) at its base and largest extra, 258 also as 284 + 31,
    and every distance symbol up to 32 768"""
    rng = np.random.default_rng(seed)
    w = Writer()
    w.fixed([rng.integers(0, 256, 33_000, dtype=np.uint8).tobytes()])
    while len(w.plain) < size:
        tokens = []
        for k in range(29):
            for n in (LEN_BASE[k], LEN_BASE[k] + (1 << LEN_EXTRA[k]) - 1):
                dk = int(rng.integers(0, 30))
                d = DIST_BASE[dk] + int(rng.integers(0, 1 << DIST_EXTRA[dk]))
                tokens += [(n, d), int(rng.integers(0, 256))]
        tokens += [(258, 32768, True), (258, 32768), (258, 1, True), (258, 24577, True)]
        w.fixed(tokens)
    w.fixed([], final=True)
    return Case("fixed_long", w, split_points=False)


def rle_258(size: int, seed: int) -> Case:
    """length-258 copies at distances 1 and 2, half of them as 284 + 31"""
    rng = np.random.default_rng(seed)
    w = Writer()
    first = True
    while len(w.plain) < size:
        tokens = [rng.integers(0, 256, 16 if first else 2, dtype=np.uint8).tobytes()]
        tokens += [(258, 1 + (j // 50) % 2, j % 2 == 0) for j in range(min(4000, (size - len(w.plain)) // 258 + 1))]
        w.dynamic(tokens, *_freq_lengths(tokens))
        first = False
    w.fixed([], final=True)
    return Case("rle_258", w, split_points=False)   # a few hundred bytes per MB: too short to cut


def header_straddle(size: int, seed: int) -> Case:
    """many dynamic blocks with the longest headers (HCLEN 19, no repeat codes, 316 code lengths) at every bit phase
    and many offsets, so that headers straddle staging and wave boundaries"""
    rng = np.random.default_rng(seed)
    w = Writer()
    while len(w.plain) < size:
        n = int(rng.integers(0, 4_000))
        tokens = [rng.integers(0, 256, n, dtype=np.uint8).tobytes()]
        if w.plain:
            tokens += [(int(rng.integers(3, 259)), int(rng.integers(1, min(len(w.plain), 32768) + 1)))]
        w.dynamic(tokens, random_lengths(286, rng), random_lengths(30, rng), hlit=286, hdist=30, hclen=19, runs="none")
    w.fixed([], final=True)
    return Case("header_straddle", w)


def hdist32_unused(size: int, seed: int) -> Case:
    """HDIST 32 with codes for distance symbols 30 and 31 that are never used: zlib rejects the header ('too many
    length or distance symbols'); the reference only rejects the symbols when they occur, so the oracle decodes it"""
    rng = np.random.default_rng(seed)
    w = Writer()
    while len(w.plain) < size:
        tokens = [rng.integers(0, 256, 20_000, dtype=np.uint8).tobytes()]
        tokens += [(int(rng.integers(3, 259)), int(rng.integers(1, min(len(w.plain) + 20_000, 32768) + 1))) for _ in range(50)]
        w.dynamic(tokens, random_lengths(286, rng), [5] * 32, hlit=286, hdist=32)
    w.fixed([], final=True)
    # (block_search takes no header with HDIST > 30 for a split point: such a stream is decoded whole)
    return Case("hdist32_unused", w, zlib_agrees=False, split_points=False)


# invalid streams: a valid prefix of `size` bytes (so that a block-parallel engine meets the defect mid-stream), then the
# defective block
def _prefix(size: int, rng) -> Writer:
    w = Writer()
    while len(w.plain) < size:
        lits = rng.integers(0, 256, min(30_000, size), dtype=np.uint8).tobytes()
        reach = min(len(w.plain) + len(lits), 32768)
        tokens = [lits] + [(int(rng.integers(3, 259)), int(rng.integers(1, reach + 1))) for _ in range(30)]
        w.dynamic(tokens, *_freq_lengths(tokens))
    return w


def _bad(name, status, err, build, prefix_cap=None):
    def make(size: int, seed: int) -> Case:
        rng = np.random.default_rng(seed)
        w = _prefix(min(size, prefix_cap or size), rng)
        build(w, rng)
        return Case(name, w, status=status, err=err)
    make.__name__ = name
    return make


def _lits(rng):
    return rng.integers(0, 256, 500, dtype=np.uint8).tobytes()


def _lit_oversubscribed(w, rng):
    lit = random_lengths(286, rng)
    lit[max((s for s in range(286) if lit[s] > 1), key=lambda s: lit[s])] -= 1
    w.dynamic([_lits(rng)], lit, random_lengths(30, rng), final=True)


def _lit_incomplete(w, rng):
    lit = random_lengths(286, rng)
    lit[min((s for s in range(286) if lit[s] < 15), key=lambda s: lit[s])] += 1
    w.dynamic([_lits(rng)], lit, random_lengths(30, rng), final=True)


def _header_defect(defect):
    def build(w, rng):
        w.dynamic([_lits(rng)], random_lengths(286, rng), random_lengths(30, rng), defect=defect, final=True)
    return build


def _hlit(n):
    def build(w, rng):
        w.dynamic([_lits(rng)], random_lengths(n, rng), random_lengths(30, rng), hlit=n, final=True)
    return build


def _hdist_used(n):
    def build(w, rng):
        dist = [5] * 32 if n == 32 else [4] + [5] * 30     # complete codes, so that the tree itself is valid
        w.dynamic([_lits(rng), ("dsym", n - 1)], random_lengths(286, rng), dist, hlit=286, hdist=n, final=True)
    return build


def _fixed_symbol(token):
    def build(w, rng):
        w.fixed([_lits(rng), token], final=True)
    return build


def _one_code_unassigned(w, rng):
    tokens = [_lits(rng), (3, 1)]
    lit, _ = _freq_lengths(tokens)
    w.dynamic(tokens + [("draw", 1, 1)], lit, [1], final=True)


def _distance_past_start(w, rng):
    w.fixed([(3, len(w.plain) + 1)], final=True)


CASES = {f.__name__: f for f in (far_window, sparse_trees, empty_blocks, fixed_long, rle_258, header_straddle,
                                 hdist32_unused)}
INVALID = {f.__name__: f for f in (
    _bad("bad_lit_oversubscribed", ERR_HUFFMAN_TABLE, (0, 0), _lit_oversubscribed),
    _bad("bad_lit_incomplete", ERR_HUFFMAN_TABLE, (0, 0), _lit_incomplete),
    _bad("bad_cl_oversubscribed", ERR_CODELENGTH_HUFFMAN_TABLE, (0, 0), _header_defect("cl_oversubscribed")),
    _bad("bad_first_repeat", ERR_CODELENGTH_SEQUENCE, (0, 0), _header_defect("first_repeat")),
    _bad("bad_repeat_overrun", ERR_CODELENGTH_SEQUENCE, (0, 0), _header_defect("repeat_overrun")),
    _bad("bad_hlit287", ERR_RUNLITERAL_SYMBOL_COUNT, (287, 0), _hlit(287)),
    _bad("bad_hlit288", ERR_RUNLITERAL_SYMBOL_COUNT, (288, 0), _hlit(288)),
    _bad("bad_hdist31_used", ERR_INVALID_SYMBOL, (30, 1), _hdist_used(31)),
    _bad("bad_hdist32_used", ERR_INVALID_SYMBOL, (31, 1), _hdist_used(32)),
    _bad("bad_fixed_lit286", ERR_INVALID_SYMBOL, (286, 0), _fixed_symbol(("lsym", 286))),
    _bad("bad_fixed_lit287", ERR_INVALID_SYMBOL, (287, 0), _fixed_symbol(("lsym", 287))),
    _bad("bad_fixed_dist30", ERR_INVALID_SYMBOL, (30, 1), _fixed_symbol(("dsym", 30))),
    _bad("bad_fixed_dist31", ERR_INVALID_SYMBOL, (31, 1), _fixed_symbol(("dsym", 31))),
    _bad("bad_one_code_unassigned", ERR_INVALID_SYMBOL, (0, 1), _one_code_unassigned),
    _bad("bad_distance_past_start", ERR_STRING_REFERENCE, (0, 0), _distance_past_start, prefix_cap=20_000),
)}


def build(name: str, size: int, seed: int = 0) -> Case:
    return (CASES.get(name) or INVALID[name])(size, seed)
