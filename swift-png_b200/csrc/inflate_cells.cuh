// inflate_cells.cuh -- intra-stream parallel DEFLATE inflate, third generation ("cells").
//
// Same decomposition as inflate_wave.cuh -- one CTA of 256 threads per stream, WAVES of 256 subsequences x
// 256 bits staged in shared memory, speculate / walk / chain / count exactly as there -- but the LZ77 half is
// new.  The ring kernel executed copies token by token (a lane per token, byte loops of very different
// lengths side by side, a sorted list + an "unresolved" bitmap for copies whose source was not final yet, and a
// polling sweep whose duration is the depth of the copy -> copy dependency chain: ncu r02 charged 33 % of all
// warp instructions at 4-9 active lanes and 21 % of the stall samples to that machinery).  Here a wave's output
// is an array of 16-bit CELLS in shared memory, one per output byte:
//
//      0x0000 .. 0x00ff   a final byte
//      0x0100 .. 0x80ff   "same byte as window position s", s = cell - 0x8100 in [-32768, -1] relative to the
//                         wave's first output byte (bytes earlier waves have already stored to HBM)
//      0xc000 .. 0xffff   "same byte as cell j" of this wave, j = cell & 0x3fff, always in front of the cell
//
//   E. emit     every thread decodes its share once more and only WRITES cells: a literal is its byte, an LZ77
//               copy is `run` pointer cells (no source is read, nothing waits, overlapping copies need no
//               special case: cell p points at p - dist, which is a cell of the same copy).
//   F. resolve  pointer jumping.  Each thread sweeps a contiguous chunk of cells in ascending order and replaces
//               every in-wave pointer by the cell it points at.  Within a chunk the sweep has sequential
//               semantics (the target was already swept), so after round one every surviving pointer leaves its
//               chunk, and every further round at least halves the number of chunks on a chain: two or three
//               rounds for PNG data, ceil(log2 256) + 1 at worst.  Racing reads are harmless -- any value a cell
//               ever holds is a true statement about its byte.  All lanes active, no atomics, no polling.
//   G. store    cells -> bytes, 16 per thread and step: final cells as they are, window cells gathered from the
//               stream's own output in HBM/L2 (stored by earlier waves), 16-byte coalesced stores, Adler-32 partial
//               sums from the same registers.
//
// There is no window in shared memory any more (the ring cost 64 KiB per stream): 75 KB per CTA, three CTAs per SM.
// A wave whose output does not fit the cell array is CUT at the token that would overflow it: the tokens in
// front are emitted, the next wave starts at that token, and the number of subsequences the next wave
// speculates on shrinks to what the cut wave used (it grows back by doubling), so highly compressible data costs
// idle threads, not repeated speculation.  Irregular input (invalid symbol on the chain, truncation, output
// overflow, a distance reaching in front of the output) goes to the serial decoder as before.
//
// Segment jobs (several CTAs per stream, StreamJob.symbolic): the output is 16-bit symbols in HBM, exactly as
// inflate_wave_kernel writes them (a byte, or the marker 0x8000 | index into the 32 KiB window in front of the segment).
// Cells are already symbolic inside a wave; for a segment the store phase keeps them symbolic across waves: a window cell
// becomes the symbol stored at that position earlier (a marker travels through copies like any other symbol), or a marker
// when the position lies in front of the segment.
//
// Replaces the reference's serial token loop Stream.readBlock(with:) and InflatorOut.expand
// (Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:266-381, LZ77.InflatorOut.swift:124-140),
// the window of LZ77.InflatorOut (LZ77.InflatorOut.swift:86-110) and, for zlib streams, the running
// MRC32 (Sources/LZ77/Wrappers/LZ77.MRC32.swift:26-47).
#pragma once

#include "inflate_wave.cuh"   // shared pieces: FastBits, wv_decode, wv_fast_header, StagedReader, bulk copy, Adler helpers

namespace pngb200 {

constexpr int      CL_CTAS_PER_SM = 3;
constexpr uint32_t CL_SLOTS       = 16000;                 // cell slots (16-bit), <= 16384 (14-bit cell index)
constexpr uint32_t CL_CAP         = CL_SLOTS - 16;         // largest wave output (the first slots mirror dst's 16-byte phase)
constexpr uint32_t CL_INWAVE      = 0xc000u;               // cell >= this: pointer to cell (cell & 0x3fff)
constexpr uint32_t CL_WINDOW_BIAS = 0x8100u;               // 0x100 <= cell < 0x8100: window position cell - 0x8100
constexpr uint32_t CL_MIN_SUBS    = 32;                    // a cut wave never shrinks its successor below one warp
// Token staging: the speculative decode (phase A) and the walks (phase B) leave every token they decode in a per-CTA
// scratch area in global memory (L2 resident: written and read back within one wave), 32 bits per token (run << 16 | distance, or byte << 16), so that the emit
// phase does not decode a third time -- it reads its share back.  own[t][k]: k-th token thread t decoded in its
// subsequence; walk[u][k]: k-th token of the walk that started at thread u's exit.
constexpr uint32_t CL_TCAP        = 64;                    // tokens kept per subsequence (more: the thread decodes again in emit)
constexpr uint32_t CL_WCAP        = 64;                    // tokens kept per walk
constexpr uint64_t CL_SCRATCH     = (uint64_t)WV_THREADS * (CL_TCAP + CL_WCAP) * sizeof(uint32_t);

struct ClShared {
    SerialShared ser;
    uint32_t     words[WV_SMEM_WORDS];
    uint32_t     mask[8 * WV_THREADS];          // [k][t]: token starts in bits 32k .. 32k+31 of subsequence t
    uint32_t     pf_tail[16];                   // (the bulk prefetch of the next wave's words lands in mask ++ pf_tail)
    uint32_t     exit_[WV_THREADS];
    uint32_t     wpos_[WV_THREADS];
    uint32_t     wn_[WV_THREADS];
    uint64_t     cross_[WV_THREADS];
    uint16_t     wc_[WV_THREADS];
    uint16_t     wk_[WV_THREADS];               // tokens the walk has decoded (staged in walk[u][..] up to CL_WCAP)
    uint16_t     next_[WV_THREADS];
    uint8_t      kind_[WV_THREADS];
    uint8_t      wlist[2][WV_THREADS];
    uint32_t     wcount[3];
    uint64_t     warp_sums[WV_WARPS + 1];
    uint32_t     adler_a[WV_WARPS], adler_b[WV_WARPS];
    uint32_t     exc[WV_WARPS], valid[WV_WARPS];
    uint32_t     last, term, anomaly, ticket;
    uint32_t     cut_pos, cut_out;
    uint32_t     hdr_mode, hdr_rel, hdr_ok, hdr_end, hdr_count;   // block header hand-over (see cl_header_preamble)              // a cut wave: bit position of the first token not emitted, bytes emitted
    uint64_t     cyc[12], tick;
    uint64_t     pf_bar;
    WvHeader     hdr;
    uint16_t     cells[CL_SLOTS] __align__(32);
};
static_assert(sizeof(ClShared) <= (228 * 1024 - CL_CTAS_PER_SM * 1024) / CL_CTAS_PER_SM, "CTAs per SM");
static_assert(CL_SLOTS <= 16384 && CL_SLOTS % 16 == 0, "14-bit cell index");

// Shared memory by explicit 32-bit shared-window addresses (st.shared / ld.shared / red.shared): with 80 registers
// per thread the compiler otherwise rebuilds the window base from SR_CgaCtaId inside the hot loops (an S2R at
// the top of every decode iteration), and cells must be accessed exactly as written (racing sweeps).
#ifdef PNGB200_EMU
inline void     sts16(saddr_t a, uint32_t v) { *(volatile uint16_t*)a = (uint16_t)v; }
inline uint32_t lds16(saddr_t a) { return *(volatile uint16_t*)a; }
inline void     sts32(saddr_t a, uint32_t v) { *(volatile uint32_t*)a = v; }
inline void     reds_or(saddr_t a, uint32_t v) { *(volatile uint32_t*)a |= v; }
#else
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v)
{
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((uint16_t)v) : "memory");
}
__device__ __forceinline__ uint32_t lds16(uint32_t a)
{
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v)
{
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void reds_or(uint32_t a, uint32_t v)
{
    asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
#endif
typedef saddr_t cellp_t;   // shared-window address of cells[0]

// Decode one token at the reader's position: the loop body of phases A, B and of the emit fallback.  One predicated
// body for literals and copies (a warp always holds both), and ONE rarely taken branch per table for everything that is
// not a plain root entry (subtable pointer, end of block, invalid code) -- wv_decode tests pointer and special
// separately, ~8 instructions more per token.  Returns 0, PF_EOB (consumed) or PF_BAD.  `tok` = run << 16 | distance
// for a copy (distance 1 .. 32768), byte << 16 for a literal; `nbytes`: bytes the token produces; `cp`: 1 for a copy.
__device__ __forceinline__ uint32_t cl_decode(FastBits& b, saddr_t lit, saddr_t dst, uint32_t& tok, uint32_t& nbytes, uint32_t& cp)
{
    const uint32_t bits = b.peek();
    uint32_t e = lds32(lit + ((bits & ((1u << LIT_ROOT) - 1u)) << 2));
    if (e & E_SPECIAL) {
        if ((e & (E_PTR | E_INVALID)) == E_PTR) e = lds32(lit + (((e >> 16) + bfe32(bits, LIT_ROOT, e_skip(e) - LIT_ROOT)) << 2));
        if (e & E_SPECIAL) {
            if (e & E_INVALID) return PF_BAD;
            b.skip(e_len(e));
            return PF_EOB;
        }
    }
    const uint32_t len = e & 15u, skipn = (e >> 4) & 31u;
    const uint32_t run = (e >> 16) + bfe32(bits, len, skipn - len);   // literals: width 0, value = the byte
    b.skip(skipn);
    cp = (e >> 9) & 1u;
    const uint32_t dbits = b.peek();
    uint32_t d = lds32(dst + ((dbits & ((1u << DIST_ROOT) - 1u)) << 2));   // ignored for literals
    if (d & E_SPECIAL) {
        if ((d & (E_PTR | E_INVALID)) == E_PTR) d = lds32(dst + (((d >> 16) + bfe32(dbits, DIST_ROOT, e_skip(d) - DIST_ROOT)) << 2));
        if (cp && (d & E_SPECIAL)) return PF_BAD;
    }
    const uint32_t dlen = d & 15u, dskip = (d >> 4) & 31u;
    const uint32_t dist = (d >> 16) + bfe32(dbits, dlen, dskip - dlen);
    b.skip(cp ? dskip : 0u);
    tok = run << 16 | (cp ? dist : 0u);
    nbytes = cp ? run : 1u;
    return 0;
}
__device__ __forceinline__ uint32_t tok_bytes(uint32_t v) { return (v & 0xffffu) ? v >> 16 : 1u; }

// the pointer cells of one LZ77 copy: destination slots [j, j + run), first slot of the wave `jbeg`.  Most copies in
// PNG data are 3 or 4 bytes long and lie entirely on one side of the wave's first byte: their cells are four
// predicated stores, no loop (a loop per copy ran at 6 of 32 lanes: copies of different lengths side by side).
__device__ __forceinline__ void cells_copy(cellp_t ch, uint32_t j, uint32_t run, uint32_t dist, uint32_t jbeg)
{
    const int32_t src = (int32_t)j - (int32_t)dist;                  // slot of the first source byte (may lie in front of the wave)
    const saddr_t to = ch + 2 * j;
    if (src >= (int32_t)jbeg || src + (int32_t)run <= (int32_t)jbeg) {
        // all in-wave (cell = 0xc000 + source slot) or all window (cell = 0x8100 + position relative to the wave's
        // first byte, in [-32768, -1])
        const uint32_t code = src >= (int32_t)jbeg ? CL_INWAVE + (uint32_t)src
                                                   : (uint32_t)((int32_t)CL_WINDOW_BIAS + src - (int32_t)jbeg);
        sts16(to, code);
        sts16(to + 2, code + 1);
        sts16(to + 4, code + 2);
        if (run > 3) sts16(to + 6, code + 3);
        for (uint32_t k = 4; k < run; ++k) sts16(to + 2 * k, code + k);
        return;
    }
    // the source starts in front of the wave and runs into it
    const uint32_t nwin = (uint32_t)((int32_t)jbeg - src);
    uint32_t code = (uint32_t)((int32_t)CL_WINDOW_BIAS + src - (int32_t)jbeg);
    uint32_t k = 0;
    for (; k < nwin; ++k) sts16(to + 2 * k, code + k);
    code = CL_INWAVE + (uint32_t)src;
    for (; k < run; ++k) sts16(to + 2 * k, code + k);
}

// ---- block header: the code lengths of a dynamic block, decoded by the whole CTA ----
// wv_fast_header leaves the ~300 code-length symbols of a dynamic header to one lane (a dependent chain of table
// look-ups: ~100 cycles per symbol, ~25 K cycles per block with seven warps waiting).  Here the part in front of them
// (block type, counts, the code-length code and its table) stays with warp 0, then
//   1. every thread decodes the symbol that WOULD start at each of its bit positions (all positions the lengths can
//      occupy, <= CL_HDR_POS): advance, number of lengths it stands for, their value -> one word per position;
//   2. one thread follows the chain of those words from the first position (one shared-memory load per symbol on
//      the critical path, nothing else) and lists the symbols it passes with their output index;
//   3. every thread expands its part of that list into the length array.
// Anything irregular -- an invalid code, a repeat without a predecessor, too many lengths, a header that runs past
// the staged words or the input -- makes the caller run parse_block_header, which owns the reference's error semantics
// (Stream.readBlockMetadata / readBlockTables, LZ77.InflatorBuffers.Stream.swift:59-263).
constexpr uint32_t CL_HDR_POS = 4480;   // 316 lengths x (7-bit code + 7 extra bits) at most, rounded up

// warp 0.  Returns 0: use the slow parser; 1: `out` is complete (stored or fixed block); 2: dynamic block, the meta table
// is built and the code lengths start at staged bit `rel_out`
template <class Shared>
__device__ int cl_header_preamble(Shared& sh, uint64_t hbase_bit, uint64_t pos, uint64_t total_bits, int lane, WvHeader& out,
                                  uint32_t& rel_out)
{
    const uint32_t* const W = sh.words;
    auto get = [&](uint32_t rel, uint32_t n) -> uint32_t {
        const uint32_t w = rel >> 5;
        const uint32_t v = __funnelshift_r(W[w], W[w + 1], rel & 31u);
        return n >= 32 ? v : v & ((1u << n) - 1u);
    };
    uint32_t rel = (uint32_t)(pos - hbase_bit);
    if (pos + 3 > total_bits) return 0;
    const uint32_t h3 = get(rel, 3);
    rel += 3;
    out.status = PNGB200_OK;
    out.final = (int32_t)(h3 & 1u);
    out.type = (int32_t)(h3 >> 1);
    out.stored = 0;
    out.nlit = out.ndist = 0;
    if (out.type == 3) return 0;
    if (out.type == 0) {
        const uint64_t boundary = (pos + 3 + 7) & ~(uint64_t)7;
        if (boundary + 32 > total_bits) return 0;
        const uint32_t v = get((uint32_t)(boundary - hbase_bit), 32);
        const uint32_t l = v & 0xffffu, m = v >> 16;
        if (l != (~m & 0xffffu)) return 0;
        out.stored = l;
        out.pos = boundary + 32;
        return 1;
    }
    uint8_t* const lens = sh.ser.lens;
    if (out.type == 1) {
        for (int k = lane; k < 320; k += 32) lens[k] = k < 144 ? 8 : k < 256 ? 9 : k < 280 ? 7 : k < 288 ? 8 : 5;
        out.nlit = 288;
        out.ndist = 32;
        out.pos = pos + 3;
        __syncwarp();
        return 1;
    }
    if (pos + 17 > total_bits) return 0;
    const uint32_t v = get(rel, 14);
    rel += 14;
    const int nlit = 257 + (int)(v & 31u), ndist = 1 + (int)((v >> 5) & 31u), nclen = 4 + (int)(v >> 10);
    if (nlit > 286) return 0;
    if (lane < 19) lens[lane] = 0;
    __syncwarp();
    if (lane < nclen) lens[c_clen_order[lane]] = (uint8_t)get(rel + 3u * (uint32_t)lane, 3);
    rel += 3u * (uint32_t)nclen;
    __syncwarp();
    build_table<META_ROOT, META_CAP>(sh.ser.meta, lens, 19, ALPHA_META, &sh.ser.scratch, lane, 32);
    if (sh.ser.scratch.status) return 0;
    __syncwarp();
    if (rel + CL_HDR_POS + 64 > 32u * WV_HDR_WORDS) return 0;   // (cannot happen: the header starts in the first staged word)
    out.nlit = nlit;
    out.ndist = ndist;
    rel_out = rel;
    return 2;
}

__global__ void __launch_bounds__(WV_THREADS, CL_CTAS_PER_SM) inflate_cells_kernel(WvParams P)
{
    PNGB200_DYN_SMEM(cl_smem);
    ClShared& sh = *reinterpret_cast<ClShared*>(cl_smem);
    const uint32_t t    = threadIdx.x;
    const unsigned lane = lane_id(), warp = t >> 5;
    if (t == 0) mbar_init(&sh.pf_bar, 1);
    static_assert(offsetof(ClShared, pf_tail) == offsetof(ClShared, mask) + sizeof(uint32_t) * 8 * WV_THREADS &&
                  sizeof(uint32_t) * WV_PF_WORDS <= sizeof(uint32_t) * (8 * WV_THREADS + 16), "prefetch area = mask ++ pf_tail");
    static_assert(offsetof(ClShared, mask) % 16 == 0 && offsetof(ClShared, cells) % 32 == 0, "alignment");
    uint32_t pf_parity = 0;
    const saddr_t sbase = opaque(smem_addr(cl_smem));
    const saddr_t words_addr = sbase + offsetof(ClShared, words);
    const saddr_t lit = sbase + offsetof(ClShared, ser) + offsetof(SerialShared, lit);
    const saddr_t dstt = sbase + offsetof(ClShared, ser) + offsetof(SerialShared, dist);
    const saddr_t mk_t = sbase + offsetof(ClShared, mask) + 4 * t;     // my column of the token-start maps: word k at + 1024 k
    const saddr_t mk_0 = sbase + offsetof(ClShared, mask);
    uint32_t* const mk = sh.mask;
    cellp_t const ch = sbase + offsetof(ClShared, cells);
    uint32_t* const tok_own  = reinterpret_cast<uint32_t*>(P.scratch + blockIdx.x * P.scratch_stride);
    uint32_t* const tok_walk = tok_own + WV_THREADS * CL_TCAP;
    uint32_t* const tok_mine = tok_own + t * CL_TCAP;

    for (;;) {
        __syncthreads();
        if (t == 0) {
            sh.ticket = atomicAdd(P.ticket, 1u);
            sh.anomaly = 0;
            for (int k = 0; k < 12; ++k) sh.cyc[k] = 0;
            sh.tick = (uint64_t)clock64();
        }
        __syncthreads();
        if (sh.ticket >= (uint32_t)P.count) return;
        const int       j   = P.order ? (int)P.order[sh.ticket] : (int)sh.ticket;
        const StreamJob job = P.jobs[j];
        StreamResult*   r   = P.results + j;

        BitReader br;
        br.init(job.src, job.src_len, job.start_bit);
        uint64_t out    = job.start_out;
        uint32_t blocks = 0, waves = 0, sweep_rounds = 0, cuts = 0;
        uint64_t n_tokens = 0, n_matches = 0, walk_tokens = 0;
        int      st     = PNGB200_OK;
        uint32_t phase  = (uint32_t)job.phase;
        uint64_t resume_bit = job.start_bit, resume_out = job.start_out;
        uint8_t* const dst = job.dst;
        const bool     sym = job.symbolic != 0;       // segment: dst is uint16_t[dst_cap]
        uint16_t* const dst16 = reinterpret_cast<uint16_t*>(job.dst);
        bool fallback = false;
        bool     pf_pending = false;
        uint64_t pf_first = 0;
        uint32_t nsub = WV_THREADS;             // subsequences the next wave speculates on
        const bool adler_on = job.start_out == 0 && !sym;
        uint32_t   s1 = 1, s2 = 0;
        uint64_t   pend_len = 0;
        bool       pend = false;
        auto fold_adler = [&]() {
            if (pend && t == 0) {
                uint64_t A = 0, B = 0;
                for (int w = 0; w < WV_WARPS; ++w) { A += sh.adler_a[w]; B += sh.adler_b[w]; }
                s2 = (uint32_t)((s2 + (pend_len % ADLER_MOD32) * s1 + B) % ADLER_MOD32);
                s1 = (uint32_t)((s1 + A) % ADLER_MOD32);
            }
            pend = false;
        };
        auto adler_hbm = [&](const uint8_t* p, uint64_t n) {
            uint64_t a = 0, bw = 0;
            const uint64_t per = (n + WV_THREADS - 1) / WV_THREADS;
            const uint64_t lo = min((uint64_t)t * per, n), hi = min(lo + per, n);
            adler_bytes(p + lo, hi - lo, n - lo, a, bw);
            uint32_t a32 = (uint32_t)(a % ADLER_MOD32), b32 = (uint32_t)(bw % ADLER_MOD32);
            for (int o = 16; o; o >>= 1) {
                a32 += __shfl_down_sync(0xffffffffu, a32, o);
                b32 += __shfl_down_sync(0xffffffffu, b32, o);
            }
            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
            pend = true;
            pend_len = n;
        };
        auto tick = [&](int i) {
            if (t == 0) {
                const uint64_t now = (uint64_t)clock64();
                sh.cyc[i] += now - sh.tick;
                sh.tick = now;
            }
        };

        if (phase == 0) {
            st = read_stream_header(br, job.format, r);
            if (st == PNGB200_OK) {
                resume_bit = br.at();
                phase = 1;
            }
        }
        if (st == PNGB200_OK && phase == 2) st = read_trailer(br, job.format, r);

        while (st == PNGB200_OK && phase == 1) {
            __syncthreads();
            fold_adler();
            {
                const uint64_t hbase = br.pos >> 5;
                for (uint32_t k = t; k < WV_HDR_WORDS; k += WV_THREADS) sh.words[k] = br.load_word(hbase + k);
                __syncthreads();
                auto slow_header = [&](WvHeader& h) {   // warp 0: the general parser, exact error semantics
                    int      type0 = 0, final0 = 0, nlit0 = 0, ndist0 = 0;
                    uint32_t stored0 = 0;
                    StagedReader sr;
                    sr.init(sh.words, hbase << 5, br.total_bits, br.pos);
                    int st0 = parse_block_header(sr, &sh.ser, r, (int)lane, &type0, &final0, &stored0, &nlit0, &ndist0);
                    h = WvHeader{st0, type0, final0, nlit0, ndist0, stored0, sr.pos};
                };
                if (warp == 0) {
                    WvHeader h;
                    uint32_t rel = 0;
                    const int mode = cl_header_preamble(sh, hbase << 5, br.pos, br.total_bits, (int)lane, h, rel);
                    if (mode == 0) slow_header(h);
                    if (lane == 0) {
                        sh.hdr = h;
                        sh.hdr_mode = (uint32_t)mode;
                        sh.hdr_rel = rel;
                    }
                }
                __syncthreads();
                if (sh.hdr_mode == 2) {
                    // ---- the code lengths of a dynamic block, by the whole CTA (tab[] and the symbol list live in the
                    //      cell array, which is idle between blocks) ----
                    const uint32_t rel = sh.hdr_rel;
                    const int      total_lens = sh.hdr.nlit + sh.hdr.ndist;
                    const saddr_t  tab = ch, list = ch + 4 * CL_HDR_POS;
                    const uint32_t* const W = sh.words;
                    for (uint32_t q = t; q < CL_HDR_POS; q += WV_THREADS) {
                        const uint32_t at = rel + q;
                        const uint32_t bits = __funnelshift_r(W[at >> 5], W[(at >> 5) + 1], at & 31u);
                        const uint32_t e = sh.ser.meta[bits & (META_CAP - 1)];
                        uint32_t word = 0;                                  // advance 0: not a symbol
                        if (!(e & E_SPECIAL)) {
                            const uint32_t len = e & 15u, sym = e >> 16, x = bits >> len;
                            // advance | lengths it stands for << 8 | value << 16 (0xff: the previous length)
                            word = sym < 16   ? (len | 1u << 8 | sym << 16)
                                 : sym == 16 ? ((len + 2u) | (3u + (x & 3u)) << 8 | 0xffu << 16)
                                 : sym == 17 ? ((len + 3u) | (3u + (x & 7u)) << 8)
                                             : ((len + 7u) | (11u + (x & 127u)) << 8);
                        }
                        sts32(tab + 4 * q, word);
                    }
                    __syncthreads();
                    if (t == 0) {
                        uint32_t p = 0, have = 0, prev = 0, count = 0, ok = 1;
                        while (have < (uint32_t)total_lens) {
                            const uint32_t e = lds32(tab + 4 * p);
                            const uint32_t adv = e & 0xffu, cnt = (e >> 8) & 0xffu;
                            uint32_t val = e >> 16;
                            if (adv == 0 || (val == 0xffu && have == 0) || have + cnt > (uint32_t)total_lens) { ok = 0; break; }
                            if (val == 0xffu) val = prev;
                            sts32(list + 4 * count, have | cnt << 9 | val << 17);
                            ++count;
                            prev = val;
                            have += cnt;
                            p += adv;
                            if (p >= CL_HDR_POS) { ok = 0; break; }
                        }
                        const uint64_t end = (hbase << 5) + rel + p;
                        if (end > br.total_bits) ok = 0;
                        sh.hdr_ok = ok;
                        sh.hdr_count = count;
                        sh.hdr.pos = end;
                    }
                    __syncthreads();
                    if (sh.hdr_ok) {
                        const uint32_t count = sh.hdr_count;
                        for (uint32_t i = t; i < count; i += WV_THREADS) {
                            const uint32_t e = lds32(list + 4 * i);
                            const uint32_t at = e & 0x1ffu, cnt = (e >> 9) & 0xffu, val = e >> 17;
                            for (uint32_t k = 0; k < cnt; ++k) sh.ser.lens[at + k] = (uint8_t)val;
                        }
                    } else if (warp == 0) {
                        WvHeader h;
                        slow_header(h);
                        if (lane == 0) sh.hdr = h;
                    }
#if defined(PNGB200_EMU) && defined(WV_PROFILE)
                    if (t == 0) wv_profile().thread_iters[5] += sh.hdr_ok ? 1 : 0, wv_profile().thread_iters[6] += sh.hdr_ok ? 0 : 1;
#endif
                }
            }
            __syncthreads();
            const WvHeader hdr = sh.hdr;
            st = hdr.status;
            if (st != PNGB200_OK) break;
            const int      type = hdr.type, final = hdr.final;
            const uint32_t stored = hdr.stored;
            br.seek(hdr.pos);
            if (type != 0) {
                st = build_block_tables(&sh.ser, r, hdr.nlit, hdr.ndist, (int)t, WV_THREADS);
                if (st != PNGB200_OK) break;
            }
            tick(0);
            if (type == 0) {
                if (!br.have(8 * (uint64_t)stored)) { st = PNGB200_NEED_MORE_INPUT; break; }
                if (out + stored > job.dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
                const uint8_t* s = job.src + (br.at() >> 3);
                if (sym) for (uint32_t k = t; k < stored; k += WV_THREADS) dst16[out + k] = s[k];
                else for (uint32_t k = t; k < stored; k += WV_THREADS) dst[out + k] = s[k];
                if (adler_on && stored) adler_hbm(s, stored);
                out += stored;
                br.seek(br.pos + 8 * (uint64_t)stored);
                __syncthreads();
                fold_adler();
                tick(9);
            } else {
                bool block_done = false;
                while (!block_done) {
                    ++waves;
                    const uint32_t wave_bits = nsub * WV_SUB_BITS;
                    // ---- stage the wave's bits in shared memory ----
                    const uint64_t wstart = br.pos;
                    const uint64_t wbase  = (wstart >> 5) & ~(uint64_t)7;
                    __syncthreads();
                    bool staged = false;
                    if (pf_pending) {
                        while (!mbar_try_wait(&sh.pf_bar, pf_parity)) {}
                        pf_parity ^= 1;
                        pf_pending = false;
                        if (wbase >= pf_first && wbase - pf_first < 4) {
                            const uint32_t* lin = sh.mask + (uint32_t)(wbase - pf_first);
                            for (uint32_t k = t; k < WV_WORDS; k += WV_THREADS) sh.words[k + (k >> 3)] = lin[k];
                            staged = true;
                        }
                    }
                    if (!staged)
                        for (uint32_t k = t; k < WV_WORDS; k += WV_THREADS)
                            sh.words[k + (k >> 3)] = br.load_word(wbase + k);
                    if (t == 0) {
                        sh.wcount[0] = 0;
                        sh.cut_pos = 0xffffffffu;
                    }
                    __syncthreads();                                      // (1)
                    fold_adler();
                    tick(1);
                    const uint32_t rel0  = (uint32_t)(wstart - (wbase << 5));  // < 256
                    const uint32_t base  = t * WV_SUB_BITS;
                    const uint32_t limit = base + WV_SUB_BITS;

                    // ---- A. speculative decode of my subsequence: token-start map, checkpoints, totals ----
                    uint32_t nout = 0, ncopy = 0, flags = 0, exit_bit = base;
                    uint32_t n = 0;                 // tokens of my own decode (staged in tok_own[t][..] up to CL_TCAP)
                    {
#pragma unroll
                        for (int k = 0; k < 8; ++k) sts32(mk_t + 1024 * k, 0);
                        if (t < nsub) {
                            FastBits b;
                            b.init(words_addr, t == 0 ? rel0 : base);
                            while (b.pos < limit) {
                                const uint32_t rr = b.pos - base;
                                reds_or(mk_t + ((rr >> 5) << 10), 1u << (rr & 31));     // this position starts a token
                                uint32_t tok = 0, nb = 0, cp = 0;
                                const uint32_t s = cl_decode(b, lit, dstt, tok, nb, cp);
                                if (s) { flags = s; break; }
                                if (n < CL_TCAP) tok_mine[n] = tok;
                                nout += nb;
                                ncopy += cp;
                                ++n;
                            }
                            exit_bit = b.pos;
                        } else {
                            flags = PF_BAD;       // not part of this wave: never reached by the chain
                        }
                        WV_COUNT(0, n);
                    }
                    sh.exit_[t] = exit_bit;
                    sh.cross_[t] = 0;
                    __syncthreads();                                      // (2) maps complete
                    tick(2);

                    // ---- B. walks (as in inflate_wave_kernel) ----
                    {
                        uint32_t u = t, pos = exit_bit, wn = 0, wc = 0, wk = 0;
                        bool     active = flags == 0;
                        sh.wk_[t] = 0;
                        if (!active) {
                            sh.kind_[t] = (uint8_t)(flags == PF_EOB ? WK_OWN_EOB : WK_OWN_BAD);
                            sh.wpos_[t] = exit_bit;
                            sh.wn_[t] = 0;
                            sh.wc_[t] = 0;
                        }
                        for (uint32_t round = 0;; ++round) {
                            const uint32_t K = WV_WALK_K << min(round, 6u);
                            bool     still = false;
                            uint32_t iters = 0;
                            if (active) {
                                FastBits b;
                                b.init(words_addr, pos);
                                uint32_t kind = WK_RUNNING;
                                const uint32_t first_sub = sh.exit_[u] >> 8;
                                bool     crossed = sh.cross_[u] != 0;
                                for (; iters < K; ++iters) {
                                    const uint32_t p = b.pos;
                                    if (p >= wave_bits) { kind = WK_END; break; }
                                    const uint32_t s = p >> 8, rr = p & 255u;
                                    if (!crossed && s > first_sub) {
                                        // (bits 32..39: walk tokens in front of the crossing, 255 = more than the staging keeps)
                                        sh.cross_[u] = 1ull << 63 | (uint64_t)p << 40 | (uint64_t)min(wk, 255u) << 32 |
                                                       (uint64_t)(wc & 0xffu) << 24 | (wn & 0xffffffu);
                                        crossed = true;
                                    }
                                    if ((lds32(mk_0 + (((rr >> 5) << 10) + (s << 2))) >> (rr & 31)) & 1u) { kind = WK_SYNC; break; }
                                    uint32_t tok = 0, nb = 0, cp = 0;
                                    const uint32_t e = cl_decode(b, lit, dstt, tok, nb, cp);
                                    if (e) { kind = e == PF_EOB ? WK_EOB : WK_BAD; break; }
                                    if (wk < CL_WCAP) tok_walk[u * CL_WCAP + wk] = tok;
                                    ++wk;
                                    wn += nb;
                                    wc += cp;
                                }
                                sh.wpos_[u] = b.pos;
                                sh.wn_[u]   = wn;
                                sh.wc_[u]   = (uint16_t)wc;
                                sh.wk_[u]   = (uint16_t)min(wk, 0xffffu);
                                sh.kind_[u] = (uint8_t)kind;
                                still = kind == WK_RUNNING;
                                walk_tokens += iters;
                            }
                            WV_COUNT(1, iters);
                            if (t == 0) sh.wcount[(round + 1) % 3] = 0;
                            const unsigned bal = __ballot_sync(0xffffffffu, still);
                            if (still) {
                                uint32_t at = 0;
                                const int leader = __ffs((int)bal) - 1;
                                if ((int)lane == leader) at = atomicAdd(&sh.wcount[round % 3], (uint32_t)__popc(bal));
                                at = __shfl_sync(bal, at, leader);
                                sh.wlist[round & 1][at + __popc(bal & ((1u << lane) - 1u))] = (uint8_t)u;
                            }
                            __syncthreads();
                            const uint32_t cnt = sh.wcount[round % 3];
                            if (cnt == 0) break;
                            active = t < cnt;
                            if (active) {
                                u   = sh.wlist[round & 1][t];
                                pos = sh.wpos_[u];
                                wn  = sh.wn_[u];
                                wc  = sh.wc_[u];
                                wk  = sh.wk_[u];
                            }
                        }
                    }
                    tick(3);
                    const uint32_t kind = sh.kind_[t], wpos = sh.wpos_[t];
                    {
                        const bool joins_next = kind == WK_SYNC && (wpos >> 8) == t + 1;
                        sh.next_[t] = (uint16_t)(kind == WK_SYNC ? wpos >> 8 : 0xffffu);
                        const unsigned e = __ballot_sync(0xffffffffu, !joins_next);
                        if (lane == 0) sh.exc[warp] = e;
                    }
                    __syncthreads();                                      // (3)

                    // ---- C. the true chain: orbit of thread 0 ----
                    if (t == 0) {
                        uint32_t E[WV_WARPS];
#pragma unroll
                        for (int w = 0; w < WV_WARPS; ++w) E[w] = sh.exc[w];
                        uint32_t cur = 0, x = 0;
                        bool     done = false;
#pragma unroll
                        for (int w = 0; w < WV_WARPS; ++w) {
                            uint32_t v = 0;
                            while (!done && cur < 32u * (w + 1)) {
                                const uint32_t lo = cur - 32u * w;
                                const uint32_t m = E[w] & (~0u << lo);
                                if (m == 0) {
                                    v |= ~0u << lo;
                                    cur = 32u * (w + 1);
                                    break;
                                }
                                const uint32_t b = (uint32_t)__ffs((int)m) - 1;
                                x = 32u * w + b;
                                v |= bit_mask(lo, b + 1);
                                const uint32_t nx = sh.next_[x];
                                if (nx == 0xffffu) done = true;
                                else cur = nx;
                            }
                            sh.valid[w] = v;
                        }
                        sh.last = x;
                        sh.term = sh.kind_[x];
                    }
                    __syncthreads();                                      // (4)
                    tick(4);

                    // ---- D. my share of the chain ----
                    const bool     on_chain = (sh.valid[warp] >> lane) & 1u;
                    const uint32_t last = sh.last, term = sh.term;
                    uint32_t from = rel0, to = exit_bit;
                    uint32_t my_nout = 0, my_ncopy = 0;
                    bool     adopted = false;
                    // my share as staged tokens: walk tokens [a_lo, a_hi) of thread a_src, then my own tokens [b_lo, n),
                    // then (last thread of the chain) my own walk's tokens; `kept`: all of them were kept by the staging
                    uint32_t a_src = 0, a_lo = 0, a_hi = 0, b_lo = 0, b_hi = 0, c_hi = 0;
                    bool     kept = true;
                    if (on_chain) {
                        uint32_t pn = 0, pc = 0, pre_n = 0, pre_c = 0;
                        b_hi = n;
                        kept = n <= CL_TCAP;
                        if (t > 0) {
                            uint32_t w = warp, m = sh.valid[w] & ((1u << lane) - 1u);
                            while (m == 0) m = sh.valid[--w];
                            const uint32_t pred = w * 32 + 31 - (uint32_t)__clz((int)m);
                            const uint32_t p0 = sh.wpos_[pred];
                            from = sh.exit_[pred];
                            pn = sh.wn_[pred];
                            pc = sh.wc_[pred];
                            a_src = pred;
                            a_hi = sh.wk_[pred];
                            kept = kept && a_hi <= CL_WCAP;
                            if (pred + 1 < t) {
                                const uint64_t cr = sh.cross_[pred];
                                if (cr) {
                                    from = (uint32_t)(cr >> 40) & 0x1ffffu;
                                    pn -= (uint32_t)cr & 0xffffffu;
                                    pc -= (uint32_t)(cr >> 24) & 0xffu;
                                    a_lo = (uint32_t)(cr >> 32) & 0xffu;
                                    kept = kept && a_lo != 255u;
                                }
                            }
                            const uint32_t rr = p0 - base, q = rr >> 5;
                            // my tokens in front of p0 (the garbage prefix) = the token starts my map holds below p0;
                            // their bytes and copies are summed from the staged tokens
                            for (uint32_t k = 0; k < q; ++k) b_lo += (uint32_t)__popc(mk[k * WV_THREADS + t]);
                            b_lo += (uint32_t)__popc(mk[q * WV_THREADS + t] & ((1u << (rr & 31)) - 1u));
                            if (b_lo <= CL_TCAP) {
                                for (uint32_t k = 0; k < b_lo; ++k) {
                                    const uint32_t v = tok_mine[k];
                                    pre_n += tok_bytes(v);
                                    pre_c += (v & 0xffffu) != 0;
                                }
                            } else {
                                FastBits b;
                                b.init(words_addr, base);
                                while (b.pos != p0 && b.pos < limit) {
                                    uint32_t tok = 0, nb = 0, cp = 0;
                                    if (cl_decode(b, lit, dstt, tok, nb, cp)) break;
                                    pre_n += nb;
                                    pre_c += cp;
                                }
                            }
                        }
                        my_nout  = pn + nout - pre_n;
                        my_ncopy = pc + ncopy - pre_c;
                        if (t == last) {
                            to = wpos;
                            my_nout += sh.wn_[t];
                            my_ncopy += sh.wc_[t];
                            c_hi = sh.wk_[t];
                            kept = kept && c_hi <= CL_WCAP;
                            if (term == WK_BAD || term == WK_OWN_BAD || (wbase << 5) + wpos > br.total_bits)
                                sh.anomaly = 1;
                        }
                    }
                    else if (t > 0 && ((sh.valid[(t - 1) >> 5] >> ((t - 1) & 31)) & 1u) && sh.kind_[t - 1] == WK_SYNC) {
                        const uint64_t cr = sh.cross_[t - 1];
                        if (cr) {
                            adopted  = true;
                            from     = sh.exit_[t - 1];
                            to       = (uint32_t)(cr >> 40) & 0x1ffffu;
                            my_nout  = (uint32_t)cr & 0xffffffu;
                            my_ncopy = (uint32_t)(cr >> 24) & 0xffu;
                            a_src    = t - 1;
                            a_hi     = (uint32_t)(cr >> 32) & 0xffu;
                            kept   = a_hi != 255u && a_hi <= CL_WCAP;
                        }
                    }
                    const uint64_t mine = (uint64_t)my_ncopy << 40 | my_nout;
                    uint64_t incl = mine;
                    for (int o = 1; o < 32; o <<= 1) {
                        uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
                        if ((int)lane >= o) incl += v;
                    }
                    if (lane == 31) sh.warp_sums[warp] = incl;
                    __syncthreads();                                      // (5)
                    if (warp == 0) {
                        uint64_t ws = lane < WV_WARPS ? sh.warp_sums[lane] : 0, wi = ws;
                        for (int o = 1; o < 32; o <<= 1) {
                            uint64_t v = __shfl_up_sync(0xffffffffu, wi, o);
                            if ((int)lane >= o) wi += v;
                        }
                        if (lane < WV_WARPS) sh.warp_sums[lane] = wi - ws;
                        if (lane == WV_WARPS - 1) sh.warp_sums[WV_WARPS] = wi;
                    }
                    __syncthreads();                                      // (6)
                    tick(5);
                    const uint64_t excl    = sh.warp_sums[warp] + incl - mine;
                    const uint64_t o64     = excl & 0xffffffffffull;
                    const uint64_t total64 = sh.warp_sums[WV_WARPS] & 0xffffffffffull;
                    const uint32_t np      = (uint32_t)(sh.warp_sums[WV_WARPS] >> 40);
                    const bool     cut     = total64 > CL_CAP;            // the wave is cut at the token that would overflow the cells
                    if (sh.anomaly || out + total64 > job.dst_cap) {
                        fallback = true;
                        break;
                    }
                    // ---- prefetch of the next wave's words (predicted start; a cut wave misses and stages directly) ----
                    if (!cut) {
                        const uint64_t nbase = wbase + wave_bits / 32;
                        const uint64_t first = nbase - ((((uintptr_t)br.words >> 2) + nbase) & 3);
                        if (first >= 1 && (first + WV_PF_WORDS + 1) * 32 <= br.total_bits) {
                            if (t == 0) {
                                fence_proxy_async();
                                mbar_expect_tx(&sh.pf_bar, sizeof(uint32_t) * WV_PF_WORDS);
                                bulk_g2s(sh.mask, br.words + first, sizeof(uint32_t) * WV_PF_WORDS, &sh.pf_bar);
                            }
                            pf_pending = true;
                            pf_first = first;
                        }
                    }
                    // ---- E. emit: decode my share once more, write cells ----
                    uint8_t* const wdst  = dst + (sym ? 2 * out : out);      // HBM address of wave offset 0
                    // slot of wave offset 0: dst's phase inside a 16-element store unit (16 bytes, or 16 symbols = 32 bytes)
                    const uint32_t shift = sym ? (uint32_t)((uintptr_t)wdst & 31) >> 1 : (uint32_t)((uintptr_t)wdst & 15);
                    // a distance may reach `reach` bytes in front of the wave (a segment: always the whole 32 KiB window)
                    const uint32_t reach = (sym || out >= WV_WINDOW) ? 0x7fffffffu : (uint32_t)out;
                    uint32_t emitted = 0, my_stop = 0xffffffffu, o = 0;
                    [[maybe_unused]] uint32_t from_staging = 0;   // (cost-model counter of emulator builds)
                    if ((on_chain || adopted) && from != to && !cut && kept) {
                        // my share was kept by the passes that decoded it: read it back (walk piece, own piece, own walk)
                        o = (uint32_t)o64;
                        bool bad_ref = false;
                        auto piece = [&](const uint32_t* p, uint32_t lo, uint32_t hi) {
                            for (uint32_t i = lo; i < hi && !bad_ref; i += 4) {
                                uint32_t tk[4];
#pragma unroll
                                for (int q = 0; q < 4; ++q) tk[q] = i + q < hi ? p[i + q] : 0u;
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    if (i + q >= hi || bad_ref) break;
                                    const uint32_t v = tk[q];
                                    const uint32_t dist = v & 0xffffu, run = v >> 16;
                                    if (dist == 0) {
                                        sts16(ch + 2 * (shift + o), run);
                                        o += 1;
                                    } else {
                                        if (dist > reach + o) { bad_ref = true; break; }
                                        cells_copy(ch, shift + o, run, dist, shift);
                                        o += run;
                                    }
                                    ++emitted;
                                }
                            }
                        };
                        piece(tok_walk + a_src * CL_WCAP, a_lo, a_hi);
                        piece(tok_mine, b_lo, b_hi);
                        piece(tok_walk + t * CL_WCAP, 0, c_hi);
                        if (bad_ref) sh.anomaly = 1;
                        from_staging = emitted;
#ifdef PNGB200_EMU
                        if (!bad_ref && o != (uint32_t)o64 + my_nout) { fprintf(stderr, "cells: kept share of thread %u is %u bytes, expected %u\n", t, o - (uint32_t)o64, my_nout); abort(); }
#endif
                    } else if ((on_chain || adopted) && from != to) {
                        if (o64 >= CL_CAP) {
                            my_stop = from;                  // nothing of my share fits
                            o = CL_CAP;                      // (if I am the first such thread, the shares in front end exactly here)
                        } else {
                            o = (uint32_t)o64;
                            bool bad_ref = false;
                            FastBits b;
                            b.init(words_addr, from);
                            while (b.pos != to && b.pos < wave_bits + 64) {
                                const uint32_t at = b.pos;
                                uint32_t tok = 0, nb = 0, cp = 0;
                                if (cl_decode(b, lit, dstt, tok, nb, cp)) break;
                                if (o + nb > CL_CAP) { my_stop = at; break; }
                                const uint32_t dist = tok & 0xffffu, run = tok >> 16;
                                if (!cp) sts16(ch + 2 * (shift + o), run);
                                else if (dist > reach + o) { bad_ref = true; break; }   // invalidStringReference: the serial decoder reports it
                                else cells_copy(ch, shift + o, run, dist, shift);
                                o += nb;
                                ++emitted;
                            }
                            if (bad_ref) sh.anomaly = 1;
                        }
                    }
                    WV_COUNT(2, emitted);
                    WV_COUNT(3, from_staging);
                    if (cut && my_stop != 0xffffffffu) atomicMin(&sh.cut_pos, my_stop);
                    __syncthreads();                                      // (7) cells written
                    tick(6);
                    if (sh.anomaly) {
                        fallback = true;
                        break;
                    }
                    uint32_t total = (uint32_t)total64;
                    if (cut) {
                        if (my_stop == sh.cut_pos) sh.cut_out = o;    // exactly one thread stopped there
                        __syncthreads();
                        total = sh.cut_out;
                        ++cuts;
                    }
                    // ---- F. resolve: pointer jumping over contiguous chunks, ascending ----
                    {
                        const uint32_t jbeg = shift, jend = shift + total;
                        const uint32_t wlo = jbeg >> 1, whi = (jend + 1) >> 1;
                        const uint32_t per = ((whi - wlo + WV_THREADS - 1) / WV_THREADS) | 1u;   // odd word stride: no bank conflicts
                        const uint32_t a = min(wlo + t * per, whi), e = min(a + per, whi);
                        uint32_t rounds = 0;
                        bool     mine = true;               // my chunk may still hold in-wave pointers
                        for (;;) {
                            bool more = false;
                            if (mine) {
                                for (uint32_t i = a; i < e; ++i) {
                                    const uint32_t w = lds32(ch + 4 * i);
                                    if ((w & (w << 1) & 0x80008000u) == 0) continue;      // no in-wave pointer in this word
                                    uint32_t c0 = w & 0xffffu, c1 = w >> 16;
                                    const bool p0 = c0 >= CL_INWAVE && 2 * i >= jbeg;
                                    const bool p1 = c1 >= CL_INWAVE && 2 * i + 1 < jend;
                                    if (p0) {
                                        // follow the chain a few hops at once: inside my chunk the first hop already lands
                                        // on a swept cell; across chunks the owner may not have got there yet
                                        c0 = lds16(ch + 2 * (c0 & 0x3fffu));
#pragma unroll 1
                                        for (int hop = 0; hop < 3 && c0 >= CL_INWAVE; ++hop) c0 = lds16(ch + 2 * (c0 & 0x3fffu));
                                        sts16(ch + 4 * i, c0);
                                        more |= c0 >= CL_INWAVE;
                                    }
                                    if (p1) {
                                        const uint32_t j1 = c1 & 0x3fffu;
                                        c1 = j1 == 2 * i ? c0 : lds16(ch + 2 * j1);
#pragma unroll 1
                                        for (int hop = 0; hop < 3 && c1 >= CL_INWAVE; ++hop) c1 = lds16(ch + 2 * (c1 & 0x3fffu));
                                        sts16(ch + 4 * i + 2, c1);
                                        more |= c1 >= CL_INWAVE;
                                    }
                                }
                                mine = more;
                            }
                            ++rounds;
                            if (!__syncthreads_or(more)) break;
                        }
                        sweep_rounds += rounds;
                        WV_COUNT(4, rounds);
                    }
                    tick(7);
                    // ---- G (segment). store: cells -> 16-bit symbols; a window cell takes the symbol stored at that position
                    //      (byte or marker), or becomes a marker when the position lies in front of the segment ----
                    if (sym && total) {
                        uint16_t* const w16   = dst16 + out;                 // symbol address of wave offset 0
                        uint16_t* const gbase = w16 - shift;                 // 32-byte aligned
                        const uint32_t end    = shift + total;               // slots [shift, end) are ours
                        auto cell_symbol = [&](uint32_t c) -> uint32_t {
                            if (c < 256u) return c;
                            const int64_t at = (int64_t)out + ((int32_t)c - (int32_t)CL_WINDOW_BIAS);   // position inside the segment
                            return at >= 0 ? (uint32_t)dst16[at] : 0x8000u | (uint32_t)(at + (int64_t)WV_WINDOW);
                        };
                        const uint32_t qlo = (shift + 15) >> 4, qhi = end >> 4;       // chunks [qlo, qhi) are whole
                        for (uint32_t c = qlo + t; c < qhi; c += WV_THREADS) {
                            const uint4 h0 = *reinterpret_cast<const uint4*>(sh.cells + (c << 4));
                            const uint4 h1 = *reinterpret_cast<const uint4*>(sh.cells + (c << 4) + 8);
                            const uint32_t hw[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
                            uint32_t v[8];
#pragma unroll
                            for (int q = 0; q < 8; ++q) v[q] = cell_symbol(hw[q] & 0xffffu) | cell_symbol(hw[q] >> 16) << 16;
                            uint4* const g = reinterpret_cast<uint4*>(gbase + (c << 4));
                            g[0] = make_uint4(v[0], v[1], v[2], v[3]);
                            g[1] = make_uint4(v[4], v[5], v[6], v[7]);
                        }
                        if (t < 2) {   // the ragged head and tail (at most 15 symbols each)
                            const uint32_t k0 = t == 0 ? shift : max(qhi << 4, shift), k1 = t == 0 ? min(qlo << 4, end) : end;
                            const bool     skip = t == 1 && qhi < qlo;
                            for (uint32_t k = k0; k < k1 && !skip; ++k) gbase[k] = (uint16_t)cell_symbol(sh.cells[k]);
                        }
                    }
                    // ---- G. store: cells -> bytes (window cells gathered from the stream's own output), 16-byte coalesced ----
                    if (!sym && total) {
                        uint8_t* const gbase = wdst - shift;                 // 16-byte aligned
                        const uint32_t end   = shift + total;                // slots [shift, end) are ours
                        uint32_t a = 0, bw = 0;
                        auto cell_byte = [&](uint32_t c) -> uint32_t {
                            // a window cell: relative position c - 0x8100 in [-32768, -1]
                            return c < 256u ? c : (uint32_t)wdst[(int32_t)c - (int32_t)CL_WINDOW_BIAS];
                        };
                        // 16 cells -> 16 bytes; the window gathers of TWO chunks are in flight before either is packed (the
                        // phase is bound by the L2 round trip of those byte loads)
                        auto fetch = [&](uint32_t lo, uint32_t (&v)[16]) {
                            const uint4 h0 = *reinterpret_cast<const uint4*>(sh.cells + lo);
                            const uint4 h1 = *reinterpret_cast<const uint4*>(sh.cells + lo + 8);
                            const uint32_t hw[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
                            for (int q = 0; q < 8; ++q) {
                                v[2 * q]     = cell_byte(hw[q] & 0xffffu);
                                v[2 * q + 1] = cell_byte(hw[q] >> 16);
                            }
                        };
                        auto pack = [&](const uint32_t (&v)[16]) -> uint4 {
                            uint32_t by[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) by[q] = v[4 * q] | v[4 * q + 1] << 8 | v[4 * q + 2] << 16 | v[4 * q + 3] << 24;
                            return make_uint4(by[0], by[1], by[2], by[3]);
                        };
                        const uint32_t qlo = (shift + 15) >> 4, qhi = end >> 4;       // chunks [qlo, qhi) are whole
                        uint32_t c = qlo + t;
                        for (; c + WV_THREADS < qhi; c += 2 * WV_THREADS) {
                            uint32_t v0[16], v1[16];
                            fetch(c << 4, v0);
                            fetch((c + WV_THREADS) << 4, v1);
                            const uint4 x0 = pack(v0), x1 = pack(v1);
                            reinterpret_cast<uint4*>(gbase)[c] = x0;
                            reinterpret_cast<uint4*>(gbase)[c + WV_THREADS] = x1;
                            adler_chunk16_u32(x0, end - (c << 4), a, bw);
                            adler_chunk16_u32(x1, end - ((c + WV_THREADS) << 4), a, bw);
                        }
                        if (c < qhi) {
                            uint32_t v0[16];
                            fetch(c << 4, v0);
                            const uint4 x0 = pack(v0);
                            reinterpret_cast<uint4*>(gbase)[c] = x0;
                            adler_chunk16_u32(x0, end - (c << 4), a, bw);
                        }
                        // the ragged head and tail (at most 15 bytes each): threads 0 and 1
                        if (t < 2) {
                            const uint32_t k0 = t == 0 ? shift : max(qhi << 4, shift), k1 = t == 0 ? min(qlo << 4, end) : end;
                            const bool     skip = t == 1 && qhi < qlo;      // (everything lies inside one chunk: thread 0 took it)
                            for (uint32_t k = k0; k < k1 && !skip; ++k) {
                                const uint32_t v = cell_byte(sh.cells[k]);
                                gbase[k] = (uint8_t)v;
                                a += v;
                                bw += (end - k) * v;
                            }
                        }
                        if (adler_on) {
                            uint32_t a32 = a, b32 = bw % ADLER_MOD32;
                            for (int o2 = 16; o2; o2 >>= 1) {
                                a32 += __shfl_down_sync(0xffffffffu, a32, o2);
                                b32 += __shfl_down_sync(0xffffffffu, b32, o2);
                            }
                            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
                            pend = true;
                            pend_len = total;
                        }
                    }
                    tick(8);
                    out += total;
                    if (t == 0) n_matches += np;
                    n_tokens += emitted;
                    if (cut) {
                        // the next wave starts at the first token that did not fit and speculates on as many
                        // subsequences as this one got through (+ a quarter), at least one warp's worth
                        const uint32_t cp = sh.cut_pos;
                        const uint32_t used = (cp >> 8) + 1;
                        nsub = min((uint32_t)WV_THREADS, max(CL_MIN_SUBS, used + (used >> 2) + 8u));
                        br.seek((wbase << 5) + cp);
                    } else {
                        nsub = min((uint32_t)WV_THREADS, nsub * 2);
                        br.seek((wbase << 5) + sh.wpos_[last]);
                        if (term == WK_EOB || term == WK_OWN_EOB) block_done = true;
                    }
                }
                if (fallback) break;
            }
            ++blocks;
            resume_bit = br.at();
            resume_out = out;
            if (job.stop_bit && !final && br.at() >= job.stop_bit) break;   // end of my segment (the host checks ==)
            if (final) {
                phase = 2;
                st = read_trailer(br, job.format, r);
                break;
            }
        }
        if (pf_pending) {
            while (!mbar_try_wait(&sh.pf_bar, pf_parity)) {}
            pf_parity ^= 1;
            pf_pending = false;
        }
        __syncthreads();
        fold_adler();
        __syncthreads();   // thread 0 has read the last piece's sums before the statistics reuse sh.adler_b
        {
            uint64_t v0 = n_tokens, v2 = walk_tokens;
            uint32_t v3 = sweep_rounds;
            for (int o = 16; o; o >>= 1) {
                v0 += __shfl_down_sync(0xffffffffu, v0, o);
                v2 += __shfl_down_sync(0xffffffffu, v2, o);
                v3 = max(v3, __shfl_down_sync(0xffffffffu, v3, o));
            }
            if (lane == 0) {
                sh.warp_sums[warp] = v0;
                sh.adler_b[warp] = (uint32_t)min(v2, (uint64_t)0xffffffffu);
                sh.exc[warp] = v3;
            }
            __syncthreads();
            if (t == 0) {
                uint64_t tk = 0, wt = 0;
                uint32_t rr = 0;
                for (int w = 0; w < WV_WARPS; ++w) {
                    tk += sh.warp_sums[w];
                    wt += sh.adler_b[w];
                    rr = max(rr, sh.exc[w]);
                }
                r->stat_waves          = waves;
                r->stat_sync_rounds    = (uint32_t)min(wt, (uint64_t)0xffffffffu);   // tokens decoded by walks
                r->stat_resolve_rounds = rr;                                          // pointer-jumping rounds
                r->stat_tokens         = tk;
                r->stat_matches        = n_matches;
                r->stat_deferred       = cuts;                                        // waves cut at the cell capacity
                for (int k = 0; k < 12; ++k) r->stat_cycles[k] = sh.cyc[k];
            }
        }
        if (fallback && sym) {
            // a segment cannot go through the byte-wise serial decoder: report it, the host decodes the stream whole
            if (t == 0) {
                r->status = PNGB200_ERR_INTERNAL;
                r->produced = out;
                r->consumed_bits = br.at();
                r->blocks = blocks;
            }
        } else if (fallback) {
            __syncthreads();
            if (warp == 0) serial_inflate(sh.ser, job, r, resume_bit, resume_out, 1, blocks);
        } else if (t == 0) {
            if (r->status == 0) r->status = st;
            r->produced      = out;
            r->consumed_bits = br.at();
            r->blocks        = blocks;
            r->resume_bit    = resume_bit;
            r->resume_out    = resume_out;
            r->phase         = phase;
            if (adler_on && job.format != PNGB200_FORMAT_GZIP) {
                const uint32_t computed = s2 << 16 | s1;
                r->checksum = computed;
                r->ck_done  = 1;
                if (r->trailer_seen && job.format != PNGB200_FORMAT_IOS && r->status >= 0 && r->declared != computed) {
                    r->status = PNGB200_ERR_STREAM_CHECKSUM;
                    r->err_a  = r->declared;
                    r->err_b  = computed;
                }
            }
        }
        if (t == 0) r->stat_fallback = fallback ? 1u : 0u;
    }
}

#ifndef PNGB200_EMU
inline int configure_inflate_cells()
{
    return (int)cudaFuncSetAttribute(inflate_cells_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(ClShared));
}
#endif

}  // namespace pngb200
