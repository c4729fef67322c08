// inflate_parallel.cuh -- intra-stream parallel DEFLATE inflate: one CTA (256 threads) per stream,
// four CTAs resident per SM so that one stream's serial stretches (header parse, fix-up rounds)
// hide behind the others' parallel ones.
//
// DEFLATE has no sync markers, but Huffman codes self-synchronise: a decoder started at a wrong
// bit offset falls into step with the true symbol sequence after a few symbols.  Per block warp 0
// parses the header, the CTA builds the decode tables (shared memory), then the block is eaten in
// WAVES of 256 subsequences x 256 bits (8 KiB of compressed data staged in shared memory, padded
// 9/8 so that lane-strided word reads are bank-conflict free):
//
//   1. sync    every thread decodes its subsequence from a guessed start (thread 0's start is
//              exact) and publishes the bit position where it crossed into the next subsequence;
//              subsequences whose predecessor's exit differs from their start are re-decoded,
//              compacted onto the lowest threads so a round costs only what it re-decodes.  The
//              verified prefix grows every round; the first end-of-block symbol on the verified
//              chain ends the wave (and the block).
//   2. scan    a CTA-wide exclusive scan of per-subsequence output byte counts.
//   3. emit    every thread decodes its subsequence once more; literals are written into a
//              shared-memory image of the wave's output (16 KiB; HBM directly if the wave expands
//              to more), every LZ77 copy becomes an item on a CTA-wide work list and its
//              destination bytes are flagged in an "unresolved" bitmap (1 bit per output byte).
//   4. resolve warps sweep the work list without CTA barriers: a copy runs as soon as none of its
//              source bytes is flagged (sources behind the wave are final by construction -- the
//              common case in PNG, where the distance is about one scanline), then clears its own
//              flags.  Time is the depth of the copy->copy dependency chain, not the copy count.
//   5. store   the shared-memory image goes to HBM with 16-byte coalesced stores.
//
// Anything unusual (invalid symbol on the verified chain, truncation, output overflow, distance
// before the start of the output) is not handled here: warp 0 re-runs the block with the serial
// decoder (inflate_serial.cuh), which owns the exact error semantics of the reference.
//
// CTAs are persistent: each takes streams from an atomic ticket (the host orders streams longest
// first), so per-CTA scratch in HBM is bounded by the number of resident CTAs.
//
// Replaces the reference's serial token loop Stream.readBlock(with:) and InflatorOut.expand
// (Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:266-381, LZ77.InflatorOut.swift:124-140).
#pragma once

#include "inflate_wave.cuh"   // shared pieces: FastBits, fast_lookup, StagedReader, wv_fast_header, CopyItem

namespace pngb200 {
namespace par {

// CTA shape (more, smaller CTAs hide each other's barrier phases)
constexpr int      PAR_THREADS      = 256;
constexpr int      PAR_CTAS_PER_SM  = 4;
constexpr int      PAR_WARPS        = PAR_THREADS / 32;
constexpr uint32_t PAR_SUB_BITS     = 256;
constexpr uint32_t PAR_SUB_WORDS    = PAR_SUB_BITS / 32;
constexpr uint32_t PAR_WAVE_WORDS   = PAR_THREADS * PAR_SUB_WORDS + 8;
constexpr uint32_t PAR_SMEM_WORDS   = PAR_WAVE_WORDS + PAR_WAVE_WORDS / 8 + 1;
constexpr uint32_t PAR_OUT_BYTES    = 16384;                         // wave output image in smem
constexpr uint32_t PAR_BITMAP_WORDS = PAR_OUT_BYTES / 32;
constexpr uint32_t PAR_LIST_CAP     = PAR_THREADS * (PAR_SUB_BITS / 2);  // >= copies per wave (2 bits min each)
constexpr uint64_t PAR_MAX_WAVE_OUT = (uint64_t)PAR_LIST_CAP * 258;

struct ParHeader {  // block header as parsed by warp 0, broadcast to the CTA
    int32_t  status, type, final, nlit, ndist;
    uint32_t stored;
    uint64_t pos;     // reader position after the header
};

struct ParShared {
    SerialShared ser;
    uint32_t     words[PAR_SMEM_WORDS];
    uint32_t     start_[PAR_THREADS];   // per subsequence: decode start (wave-relative bit)
    uint32_t     exit_[PAR_THREADS];    //                  first symbol boundary past its end
    uint32_t     nout_[PAR_THREADS];    //                  output bytes
    uint16_t     ncopy_[PAR_THREADS];   //                  LZ77 copies
    uint8_t      flag_[PAR_THREADS];    //                  PF_EOB / PF_BAD
    uint16_t     list_[PAR_THREADS];    // compacted ids of subsequences that must be re-decoded
    uint32_t     bitmap[PAR_BITMAP_WORDS];
    __align__(16) uint8_t outbuf[PAR_OUT_BYTES + 32];
    uint64_t     warp_sums[32];
    uint32_t     first_need[2], first_stop[2], nlist[2];
    uint32_t     npend, anomaly, ticket, pad;
    uint64_t     cyc[12], tick;         // phase timers (thread 0), as in inflate_wave_kernel
    // running Adler-32 of the stream (zlib / ios streams decoded from their first byte), folded wave by wave from the
    // partial sums the store phase leaves here: no second pass over the inflated bytes (as in inflate_wave_kernel)
    uint64_t     pend_len;
    uint32_t     s1, s2, pend;
    uint32_t     adler_a[PAR_WARPS], adler_b[PAR_WARPS];
    ParHeader    hdr;
};

struct ParParams {
    const StreamJob* jobs;
    StreamResult*    results;
    const uint32_t*  order;
    uint32_t*        ticket;       // global work counter (zeroed before launch)
    uint8_t*         scratch;      // per-CTA: copy list + unresolved bitmap for oversized waves
    uint64_t         scratch_stride;
    uint64_t         bitmap_words; // size of the HBM bitmap of each CTA
    int              count;
};

// sync-phase decode: symbol boundaries and output byte count only
__device__ __forceinline__ void par_decode_count(const ParShared& sh, uint32_t start, uint32_t limit,
                                                 uint32_t& exit_bit, uint32_t& nout, uint32_t& ncopy,
                                                 uint32_t& flags)
{
    FastBits b;
    // shared memory addressed from a base the compiler cannot rebuild from SR_CgaCtaId inside the loop
    const saddr_t sb = opaque(smem_addr(&sh));
    b.init(sb + offsetof(ParShared, words), start);
    const saddr_t lit = sb + offsetof(ParShared, ser) + offsetof(SerialShared, lit), dst = sb + offsetof(ParShared, ser) + offsetof(SerialShared, dist);
    nout  = 0;
    ncopy = 0;
    flags = 0;
    // literal and copy tokens run through ONE predicated body: in a warp some lanes always hold a
    // literal while others hold a copy, so two divergent paths would cost their sum every iteration
    while (b.pos < limit) {
        const uint32_t bits = b.peek();
        const uint32_t e = fast_lookup<LIT_ROOT>(lit, bits);
        if (e & E_SPECIAL) {  // end of block, or an invalid code: rare, leave the loop
            if (e & E_INVALID) flags = PF_BAD;
            else { b.skip(e_len(e)); flags = PF_EOB; }
            break;
        }
        const uint32_t len = e & 15u, skipn = (e >> 4) & 31u;
        const uint32_t run = (e >> 16) + bfe32(bits, len, skipn - len);  // literals: width 0
        b.skip(skipn);
        const uint32_t copy = e & E_COPY;
        const uint32_t d = fast_lookup<DIST_ROOT>(dst, b.peek());  // ignored for literals
        if (copy && (d & E_SPECIAL)) { flags = PF_BAD; break; }
        b.skip(copy ? (d >> 4) & 31u : 0u);
        nout += copy ? run : 1u;
        ncopy += copy >> 9;
    }
    exit_bit = (flags & PF_BAD) ? max(b.pos, limit) : b.pos;
}

// ---- unresolved-byte bitmap (bit i = output byte i of the wave is not final yet) ----
// spans of <= 33 bits touch at most two words: straight-line fast path, generic loop otherwise
__device__ __forceinline__ void bits_set(uint32_t* U, uint32_t a, uint32_t b)
{
    const uint32_t wa = a >> 5, wb = (b - 1) >> 5;
    if (wa == wb) { atomicOr(U + wa, bit_mask(a & 31, ((b - 1) & 31) + 1)); return; }
    atomicOr(U + wa, bit_mask(a & 31, 32));
    for (uint32_t w = wa + 1; w < wb; ++w) atomicOr(U + w, ~0u);
    atomicOr(U + wb, bit_mask(0, ((b - 1) & 31) + 1));
}
__device__ __forceinline__ void bits_clear(uint32_t* U, uint32_t a, uint32_t b)
{
    const uint32_t wa = a >> 5, wb = (b - 1) >> 5;
    if (wa == wb) { atomicAnd(U + wa, ~bit_mask(a & 31, ((b - 1) & 31) + 1)); return; }
    atomicAnd(U + wa, ~bit_mask(a & 31, 32));
    for (uint32_t w = wa + 1; w < wb; ++w) atomicAnd(U + w, 0u);
    atomicAnd(U + wb, ~bit_mask(0, ((b - 1) & 31) + 1));
}
__device__ __forceinline__ bool bits_all_clear(const uint32_t* U, uint32_t a, uint32_t b)
{
    const volatile uint32_t* V = U;
    const uint32_t wa = a >> 5, wb = (b - 1) >> 5;
    uint32_t any;
    if (wa == wb) any = V[wa] & bit_mask(a & 31, ((b - 1) & 31) + 1);
    else {
        any = (V[wa] & bit_mask(a & 31, 32)) | (V[wb] & bit_mask(0, ((b - 1) & 31) + 1));
        for (uint32_t w = wa + 1; w < wb; ++w) any |= V[w];
    }
    __threadfence_block();
    return any == 0;
}

// One LZ77 copy whose needed source bytes are final.  The wave's output lives at `img` (shared
// memory image, or the HBM destination itself); sources at negative wave offsets are read from
// HBM at `hbm` (= destination address of wave offset 0).
__device__ __forceinline__ void lz_copy(uint8_t* img, const uint8_t* hbm, bool img_is_hbm, uint32_t o,
                                        uint32_t run, uint32_t dist)
{
    const int64_t src = (int64_t)o - (int64_t)dist;
    uint8_t*      to  = img + o;
    if (run <= 4 && dist >= 4 && (img_is_hbm || src >= 0 || src + (int64_t)run <= 0)) {
        // the common short copy: all loads first, then the stores
        const uint8_t* from = (img_is_hbm || src < 0) ? hbm + src : img + src;
        uint8_t b0 = from[0], b1 = from[1], b2 = from[2], b3 = run == 4 ? from[3] : 0;
        to[0] = b0; to[1] = b1; to[2] = b2;
        if (run == 4) to[3] = b3;
        return;
    }
    if (img_is_hbm || src >= 0 || src + (int64_t)run <= 0) {
        const uint8_t* from = (img_is_hbm || src < 0) ? hbm + src : img + src;
        if (dist >= 4) {  // byte k+3 reads k+3-dist < k: four independent loads per step even when overlapping
            uint32_t k = 0;
            for (; k + 4 <= run; k += 4) {
                uint8_t b0 = from[k], b1 = from[k + 1], b2 = from[k + 2], b3 = from[k + 3];
                to[k] = b0; to[k + 1] = b1; to[k + 2] = b2; to[k + 3] = b3;
            }
            for (; k < run; ++k) to[k] = from[k];
        } else {
            uint32_t q = 0;
            for (uint32_t k = 0; k < run; ++k) {
                to[k] = from[q];
                if (++q == dist) q = 0;
            }
        }
    } else {
        // source starts behind the wave (HBM) and runs into the image: byte k comes from wave
        // offset src + k; offsets < 0 are in HBM, the rest were written earlier by this loop
        for (uint32_t k = 0; k < run; ++k) {
            const int64_t p = src + (int64_t)k;
            to[k] = p < 0 ? hbm[p] : img[p];
        }
    }
}

// One body, two register budgets: 4 CTAs per SM (64 registers, a few spills) when there are streams for them, 3 CTAs
// per SM (80 registers, none) when the batch only fills three slots per SM anyway -- the 444 x 8K benchmark batch.
__device__ __forceinline__ void inflate_parallel_body(ParParams P)
{
    PNGB200_DYN_SMEM(par_smem);
    ParShared& sh = *reinterpret_cast<ParShared*>(par_smem);
    const uint32_t t    = threadIdx.x;
    const unsigned lane = lane_id(), warp = t >> 5;
    CopyItem* const list    = reinterpret_cast<CopyItem*>(P.scratch + blockIdx.x * P.scratch_stride);
    uint32_t* const gbitmap = reinterpret_cast<uint32_t*>(P.scratch + blockIdx.x * P.scratch_stride +
                                                         sizeof(CopyItem) * PAR_LIST_CAP);
    for (uint32_t k = t; k < PAR_BITMAP_WORDS; k += PAR_THREADS) sh.bitmap[k] = 0;

    for (;;) {
        __syncthreads();
        if (t == 0) {
            sh.ticket = atomicAdd(P.ticket, 1u);
            sh.anomaly = 0;
            for (int k = 0; k < 12; ++k) sh.cyc[k] = 0;
            sh.tick = (uint64_t)clock64();
            sh.s1 = 1;
            sh.s2 = 0;
            sh.pend = 0;
        }
// fold the partial sums of the piece that was stored last into (s1, s2); call right after a barrier
#define PAR_FOLD_ADLER()                                                                                     \
    do {                                                                                                     \
        if (t == 0 && sh.pend) {                                                                             \
            uint64_t A_ = 0, B_ = 0;                                                                         \
            for (int w_ = 0; w_ < PAR_WARPS; ++w_) { A_ += sh.adler_a[w_]; B_ += sh.adler_b[w_]; }           \
            sh.s2 = (uint32_t)((sh.s2 + (sh.pend_len % ADLER_MOD32) * sh.s1 + B_) % ADLER_MOD32);            \
            sh.s1 = (uint32_t)((sh.s1 + A_) % ADLER_MOD32);                                                  \
            sh.pend = 0;                                                                                     \
        }                                                                                                    \
    } while (0)
// thread 0 charges the cycles since the last tick to phase i: 0 header+tables, 1 stage, 3 speculate + re-decode
// rounds, 5 scan, 6 emit, 7 resolve, 8 store
#define PAR_TICK(i)                                          \
    do {                                                     \
        if (t == 0) {                                        \
            const uint64_t now_ = (uint64_t)clock64();       \
            sh.cyc[i] += now_ - sh.tick;                     \
            sh.tick = now_;                                  \
        }                                                    \
    } while (0)
        __syncthreads();
        if (sh.ticket >= (uint32_t)P.count) return;
        const int       j   = P.order ? (int)P.order[sh.ticket] : (int)sh.ticket;
        const StreamJob job = P.jobs[j];
        StreamResult*   r   = P.results + j;

        BitReader br;
        br.init(job.src, job.src_len, job.start_bit);
        uint64_t out    = job.start_out;
        uint32_t blocks = 0, waves = 0, sync_rounds = 0, resolve_rounds = 0;
        int      st     = PNGB200_OK;
        uint32_t phase  = (uint32_t)job.phase;
        uint64_t resume_bit = job.start_bit, resume_out = job.start_out;
        uint8_t* const dst = job.dst;
        bool fallback = false;
        const bool adler_on = job.start_out == 0;   // this launch sees the stream from its first byte
        // CTA-wide partial sums of `n` finished bytes at HBM address `p` (stored blocks, oversized waves)
        auto adler_hbm = [&](const uint8_t* p, uint64_t n) {
            uint64_t a = 0, bw = 0;
            const uint64_t per = (n + PAR_THREADS - 1) / PAR_THREADS;
            const uint64_t lo = min((uint64_t)t * per, n), hi = min(lo + per, n);
            adler_bytes(p + lo, hi - lo, n - lo, a, bw);
            uint32_t a32 = (uint32_t)(a % ADLER_MOD32), b32 = (uint32_t)(bw % ADLER_MOD32);
            for (int o = 16; o; o >>= 1) {
                a32 += __shfl_down_sync(0xffffffffu, a32, o);
                b32 += __shfl_down_sync(0xffffffffu, b32, o);
            }
            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
            if (t == 0) { sh.pend = 1; sh.pend_len = n; }
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
            // warp 0 walks the header bits alone; the CTA then builds the tables together
            __syncthreads();
            PAR_FOLD_ADLER();
            {
                const uint64_t hbase = br.pos >> 5;
                for (uint32_t k = t; k < WV_HDR_WORDS; k += PAR_THREADS) sh.words[k] = br.load_word(hbase + k);
                __syncthreads();
                if (warp == 0) {
                    WvHeader h;
                    if (!wv_fast_header(sh, hbase << 5, br.pos, br.total_bits, (int)lane, h)) {
                        int      type0 = 0, final0 = 0, nlit0 = 0, ndist0 = 0;
                        uint32_t stored0 = 0;
                        StagedReader sr;
                        sr.init(sh.words, hbase << 5, br.total_bits, br.pos);
                        int st0 = parse_block_header(sr, &sh.ser, r, (int)lane, &type0, &final0, &stored0, &nlit0, &ndist0);
                        h = WvHeader{st0, type0, final0, nlit0, ndist0, stored0, sr.pos};
                    }
                    if (lane == 0) sh.hdr = ParHeader{h.status, h.type, h.final, h.nlit, h.ndist, h.stored, h.pos};
                }
            }
            __syncthreads();
            const ParHeader hdr = sh.hdr;
            st = hdr.status;
            if (st != PNGB200_OK) break;
            const int      type = hdr.type, final = hdr.final;
            const uint32_t stored = hdr.stored;
            br.seek(hdr.pos);
            if (type != 0) {
                st = build_block_tables(&sh.ser, r, hdr.nlit, hdr.ndist, (int)t, PAR_THREADS);
                if (st != PNGB200_OK) break;
            }
            PAR_TICK(0);
            if (type == 0) {
                if (!br.have(8 * (uint64_t)stored)) { st = PNGB200_NEED_MORE_INPUT; break; }
                if (out + stored > job.dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
                const uint8_t* s = job.src + (br.at() >> 3);
                for (uint32_t k = t; k < stored; k += PAR_THREADS) dst[out + k] = s[k];
                if (adler_on && stored) adler_hbm(s, stored);
                out += stored;
                br.seek(br.pos + 8 * (uint64_t)stored);
                __syncthreads();
                PAR_FOLD_ADLER();
            } else {
                bool block_done = false;
                while (!block_done) {
                    ++waves;
                    // ---- stage the wave's bits in shared memory ----
                    const uint64_t wstart = br.pos;                       // absolute bit (reader space)
                    const uint64_t wbase  = (wstart >> 5) & ~(uint64_t)7; // first staged word
                    __syncthreads();
                    PAR_FOLD_ADLER();
                    for (uint32_t k = t; k < PAR_WAVE_WORDS; k += PAR_THREADS)
                        sh.words[k + (k >> 3)] = br.load_word(wbase + k);
                    if (t == 0) {
                        sh.npend = 0;
                        sh.first_need[0] = sh.first_need[1] = PAR_THREADS;
                        sh.first_stop[0] = sh.first_stop[1] = PAR_THREADS;
                        sh.nlist[0] = sh.nlist[1] = 0;
                    }
                    __syncthreads();
                    PAR_TICK(1);
                    const uint32_t rel0  = (uint32_t)(wstart - (wbase << 5));  // < 256
                    const uint32_t limit = (t + 1) * PAR_SUB_BITS;
                    {
                        uint32_t s0 = t == 0 ? rel0 : t * PAR_SUB_BITS, ex0, n0, c0, fl0;
                        par_decode_count(sh, s0, limit, ex0, n0, c0, fl0);
                        sh.start_[t] = s0;
                        sh.exit_[t]  = ex0;
                        sh.nout_[t]  = n0;
                        sh.ncopy_[t] = (uint16_t)c0;
                        sh.flag_[t]  = (uint8_t)fl0;
                    }
                    // ---- sync rounds: only subsequences whose start moved are re-decoded, compacted
                    //      onto the lowest threads so that a round costs what it re-decodes ----
                    uint32_t nvalid = PAR_THREADS;
                    bool     stop_found = false;
                    for (uint32_t round = 0;; ++round) {
                        const uint32_t p = round & 1;
                        ++sync_rounds;
                        __syncthreads();
                        if (t == 0) {  // the other parity's counters are idle during this round
                            sh.first_need[p ^ 1] = PAR_THREADS;
                            sh.first_stop[p ^ 1] = PAR_THREADS;
                            sh.nlist[p ^ 1] = 0;
                        }
                        const uint32_t prev_exit = t > 0 ? sh.exit_[t - 1] : 0;
                        const bool need = t > 0 && prev_exit != sh.start_[t];
                        if (need) atomicMin(&sh.first_need[p], t);
                        __syncthreads();
                        const uint32_t fn = sh.first_need[p];
                        if (t < fn && sh.flag_[t] != 0) atomicMin(&sh.first_stop[p], t);
                        __syncthreads();
                        const uint32_t fs = sh.first_stop[p];
                        if (fs < PAR_THREADS) { nvalid = fs + 1; stop_found = true; break; }
                        if (fn == PAR_THREADS) break;
                        const unsigned ballot = __ballot_sync(0xffffffffu, need);
                        if (need) {
                            uint32_t base = 0;
                            const int leader = __ffs(ballot) - 1;
                            if ((int)lane == leader) base = atomicAdd(&sh.nlist[p], (uint32_t)__popc(ballot));
                            base = __shfl_sync(ballot, base, leader);
                            sh.list_[base + __popc(ballot & ((1u << lane) - 1u))] = (uint16_t)t;
                            sh.start_[t] = prev_exit;
                        }
                        __syncthreads();
                        const uint32_t cnt = sh.nlist[p];
                        if (t < cnt) {
                            const uint32_t u = sh.list_[t];
                            uint32_t ex0, n0, c0, fl0;
                            par_decode_count(sh, sh.start_[u], (u + 1) * PAR_SUB_BITS, ex0, n0, c0, fl0);
                            sh.exit_[u]  = ex0;
                            sh.nout_[u]  = n0;
                            sh.ncopy_[u] = (uint16_t)c0;
                            sh.flag_[u]  = (uint8_t)fl0;
                        }
                    }
                    __syncthreads();
                    PAR_TICK(3);
                    const uint32_t my_start = sh.start_[t], n = sh.nout_[t];
                    // ---- anomalies on the verified chain -> serial decoder ----
                    if (t == nvalid - 1 && ((sh.flag_[t] & PF_BAD) || (wbase << 5) + sh.exit_[t] > br.total_bits))
                        sh.anomaly = 1;
                    // ---- scan of output byte counts and copy counts (packed: copies << 40 | bytes) ----
                    const uint64_t mine = t < nvalid ? ((uint64_t)sh.ncopy_[t] << 40 | n) : 0;
                    uint64_t incl = mine;
                    for (int o = 1; o < 32; o <<= 1) {
                        uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
                        if ((int)lane >= o) incl += v;
                    }
                    if (lane == 31) sh.warp_sums[warp] = incl;
                    __syncthreads();
                    if (warp == 0) {
                        uint64_t ws = lane < PAR_WARPS ? sh.warp_sums[lane] : 0, wi = ws;
                        for (int o = 1; o < 32; o <<= 1) {
                            uint64_t v = __shfl_up_sync(0xffffffffu, wi, o);
                            if ((int)lane >= o) wi += v;
                        }
                        if (lane < PAR_WARPS) sh.warp_sums[lane] = wi - ws;  // exclusive
                        if (lane == PAR_WARPS - 1) sh.warp_sums[PAR_WARPS] = wi;  // wave totals
                    }
                    __syncthreads();
                    PAR_TICK(5);
                    const uint64_t excl    = sh.warp_sums[warp] + incl - mine;
                    const uint32_t o_start = (uint32_t)(excl & 0xffffffffffull);
                    uint32_t       c_next  = (uint32_t)(excl >> 40);           // my first list slot
                    const uint32_t total   = (uint32_t)(sh.warp_sums[PAR_WARPS] & 0xffffffffffull);
                    const uint32_t np      = (uint32_t)(sh.warp_sums[PAR_WARPS] >> 40);
                    if (sh.anomaly || out + total > job.dst_cap || total > P.bitmap_words * 32) {
                        fallback = true;
                        break;
                    }
                    // ---- the next wave will almost always start in the word after this one's last: ask the copy
                    //      engine to pull its 8 KiB into L2 now (bulk prefetch), so the stage phase of the next
                    //      wave does not wait for HBM ----
                    {
                        const uint64_t nbase = wbase + PAR_THREADS * PAR_SUB_WORDS;
                        const uint64_t first = nbase - ((((uintptr_t)br.words >> 2) + nbase) & 3);   // 16-byte aligned
                        if (t == 0 && first >= 1 && (first + WV_PF_WORDS + 1) * 32 <= br.total_bits) bulk_prefetch_l2(br.words + first, 4 * WV_PF_WORDS);
                    }
                    // ---- emit: literals into the output image, copies onto the work list ----
                    uint8_t* const  wdst   = dst + out;           // HBM address of wave offset 0
                    const uint32_t  shift  = (uint32_t)((uintptr_t)wdst & 15);
                    const bool      in_hbm = total > PAR_OUT_BYTES;
                    uint8_t* const  img    = in_hbm ? wdst : sh.outbuf + shift;
                    uint32_t* const U      = in_hbm ? gbitmap : sh.bitmap;
                    if (t < nvalid) {
                        FastBits b;
                        const saddr_t sb = opaque(smem_addr(&sh));   // (see par_decode_count)
                        b.init(sb + offsetof(ParShared, words), my_start);
                        const saddr_t lit = sb + offsetof(ParShared, ser) + offsetof(SerialShared, lit), dst = sb + offsetof(ParShared, ser) + offsetof(SerialShared, dist);
                        uint32_t o = o_start;
                        uint32_t mw = o_start >> 5, mbits = 0;   // pending unresolved-bit word
                        while (b.pos < limit) {
                            const uint32_t bits = b.peek();
                            const uint32_t e = fast_lookup<LIT_ROOT>(lit, bits);
                            if (e & E_SPECIAL) break;  // end of block
                            const uint32_t len = e & 15u, skipn = (e >> 4) & 31u;
                            const uint32_t run = (e >> 16) + bfe32(bits, len, skipn - len);
                            b.skip(skipn);
                            const bool     is_copy = (e & E_COPY) != 0;
                            const uint32_t dbits = b.peek();
                            const uint32_t d = fast_lookup<DIST_ROOT>(dst, dbits);
                            const uint32_t dlen = d & 15u, dskip = (d >> 4) & 31u;
                            const uint32_t dist = (d >> 16) + bfe32(dbits, dlen, dskip - dlen);
                            b.skip(is_copy ? dskip : 0u);
                            if (!is_copy) {
                                img[o++] = (uint8_t)run;  // e_value of a literal entry is the byte
                                continue;
                            }
                            if ((uint64_t)dist > out + o) {  // invalidStringReference
                                sh.anomaly = 1;
                                break;
                            }
                            // flag [o, o + run) as unresolved; words are flushed once, when left
                            for (uint32_t a = o, e2 = o + run; a < e2;) {
                                const uint32_t w = a >> 5;
                                if (w != mw) {
                                    if (mbits) atomicOr(U + mw, mbits);
                                    mw = w;
                                    mbits = 0;
                                }
                                const uint32_t hi = min(e2, (w + 1) << 5);
                                mbits |= bit_mask(a & 31, ((hi - 1) & 31) + 1);
                                a = hi;
                            }
                            list[c_next++] = CopyItem{o, run | (dist - 1) << 16};  // list is sorted by o
                            o += run;
                        }
                        if (mbits) atomicOr(U + mw, mbits);
                    }
                    __threadfence_block();
                    __syncthreads();
                    PAR_TICK(6);
                    // ---- resolve: no CTA barriers.  The list is sorted by output offset and a copy only
                    //      depends on smaller offsets, so a lane may simply block on its current item
                    //      (items t, t + 512, ... in order): the smallest open item is always ready ----
                    if (!sh.anomaly && np) {
                        // the list lives in L2: the item after the current one is fetched while the current
                        // one is being copied
                        uint32_t idx  = t;
                        CopyItem it   = CopyItem{0, 0}, nxt = CopyItem{0, 0};
                        bool     have = false, have_nxt = false;
                        if (idx < np) {
                            nxt = list[idx];
                            idx += PAR_THREADS;
                            have_nxt = true;
                        }
                        for (;;) {
                            if (!have && have_nxt) {
                                it = nxt;
                                have = true;
                                have_nxt = idx < np;
                                if (have_nxt) {
                                    nxt = list[idx];
                                    idx += PAR_THREADS;
                                }
                            }
                            bool progressed = false;
                            if (have) {
                                const uint32_t run = it.run_dist & 0xffff, dist = (it.run_dist >> 16) + 1;
                                const int64_t  src = (int64_t)it.o - (int64_t)dist;
                                const int64_t  hi  = src + (int64_t)min(run, dist);
                                bool ready = true;
                                if (hi > 0) ready = bits_all_clear(U, (uint32_t)max(src, (int64_t)0), (uint32_t)hi);
                                if (ready) {
                                    lz_copy(img, wdst, in_hbm, it.o, run, dist);
                                    __threadfence_block();
                                    bits_clear(U, it.o, it.o + run);
                                    have = false;
                                    progressed = true;
                                }
                            }
                            ++resolve_rounds;
                            if (!__any_sync(0xffffffffu, have || have_nxt)) break;
                            if (!__any_sync(0xffffffffu, progressed)) __nanosleep(40);
                        }
                    }
                    __threadfence_block();
                    __syncthreads();
                    PAR_TICK(7);
                    if (sh.anomaly) {
                        // leave the bitmap clean for whoever uses it next
                        for (uint32_t k = t; k < (total + 31) / 32; k += PAR_THREADS) U[k] = 0;
                        fallback = true;
                        break;
                    }
                    // ---- store: shared-memory image -> HBM, 16-byte coalesced ----
                    if (!in_hbm && total) {
                        uint8_t* const       base = wdst - shift;            // 16-byte aligned
                        const uint32_t       end  = shift + total;           // bytes [shift, end) are ours
                        const uint32_t       nq   = (end + 15) >> 4;
                        const uint4* const   q    = reinterpret_cast<const uint4*>(sh.outbuf);
                        uint32_t a = 0, bw = 0;   // 32 bits are enough for one thread's chunks of a 16 KiB image
                        for (uint32_t c = t; c < nq; c += PAR_THREADS) {
                            const uint32_t lo = c << 4, hi = lo + 16;
                            if (lo >= shift && hi <= end) {
                                const uint4 x = q[c];
                                reinterpret_cast<uint4*>(base)[c] = x;
                                adler_chunk16_u32(x, end - lo, a, bw);
                            } else {
                                for (uint32_t k = max(lo, shift); k < min(hi, end); ++k) {
                                    const uint8_t v = sh.outbuf[k];
                                    base[k] = v;
                                    a += v;
                                    bw += (end - k) * v;
                                }
                            }
                        }
                        if (adler_on) {
                            uint32_t a32 = a, b32 = bw % ADLER_MOD32;
                            for (int o = 16; o; o >>= 1) {
                                a32 += __shfl_down_sync(0xffffffffu, a32, o);
                                b32 += __shfl_down_sync(0xffffffffu, b32, o);
                            }
                            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
                            if (t == 0) { sh.pend = 1; sh.pend_len = total; }
                        }
                    } else if (in_hbm && adler_on && total) {
                        adler_hbm(wdst, total);
                    }
                    PAR_TICK(8);
                    out += total;
                    br.seek((wbase << 5) + sh.exit_[nvalid - 1]);
                    if (stop_found) block_done = true;
                }
                if (fallback) break;
            }
            ++blocks;
            resume_bit = br.at();
            resume_out = out;
            if (final) {
                phase = 2;
                st = read_trailer(br, job.format, r);
                break;
            }
        }
        __syncthreads();
        PAR_FOLD_ADLER();
        if (fallback) {
            // the serial decoder redoes this block (and whatever follows) and owns the result record
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
                // LZ77.InflatorBuffers.advance(.checksum): compare with the trailer (InflatorBuffers.swift:109-130)
                const uint32_t computed = sh.s2 << 16 | sh.s1;
                r->checksum = computed;
                r->ck_done  = 1;
                if (r->trailer_seen && job.format != PNGB200_FORMAT_IOS && r->status >= 0 && r->declared != computed) {
                    r->status = PNGB200_ERR_STREAM_CHECKSUM;
                    r->err_a  = r->declared;
                    r->err_b  = computed;
                }
            }
        }
        if (t == 0) {
            for (int k = 0; k < 12; ++k) r->stat_cycles[k] = sh.cyc[k];
            r->stat_waves          = waves;
            r->stat_sync_rounds    = sync_rounds;
            r->stat_resolve_rounds = resolve_rounds;
            r->stat_fallback       = fallback ? 1u : 0u;
        }
    }
}

__global__ void __launch_bounds__(PAR_THREADS, PAR_CTAS_PER_SM) inflate_parallel_kernel(ParParams P) { inflate_parallel_body(P); }
__global__ void __launch_bounds__(PAR_THREADS, 3) inflate_parallel_kernel3(ParParams P) { inflate_parallel_body(P); }

#ifndef PNGB200_EMU
// host side: opt in to the large dynamic shared memory on the current device (once per context)
inline int configure_inflate_parallel()
{
    int rc = (int)cudaFuncSetAttribute(inflate_parallel_kernel3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ParShared));
    if (rc) return rc;
    return (int)cudaFuncSetAttribute(inflate_parallel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(ParShared));
}
#endif

inline uint64_t par_bitmap_words(uint64_t max_dst_cap)
{
    uint64_t bytes = max_dst_cap < PAR_MAX_WAVE_OUT ? max_dst_cap : PAR_MAX_WAVE_OUT;
    return (bytes + 31) / 32 + 8;
}
inline uint64_t par_scratch_stride(uint64_t bitmap_words)
{
    uint64_t s = sizeof(CopyItem) * (uint64_t)PAR_LIST_CAP + 4 * bitmap_words;
    return (s + 255) / 256 * 256;
}

}  // namespace par
using par::ParParams;
using par::ParShared;
using par::inflate_parallel_kernel;
using par::inflate_parallel_kernel3;
using par::PAR_THREADS;
using par::PAR_CTAS_PER_SM;
using par::par_bitmap_words;
using par::par_scratch_stride;
#ifndef PNGB200_EMU
using par::configure_inflate_parallel;
#endif
}  // namespace pngb200
